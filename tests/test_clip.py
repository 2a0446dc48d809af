"""CLIP image towers on the CPU: the Hugging Face converter, the GGUF architecture keys, the emulation against an independent
float64 oracle (transformers' CLIPVisionModelWithProjection), and the refusals that need no GPU."""
import copy
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.util import pkg, gf, model_path
from tests import clip_oracle as co
from tests import fp8_reference as fr
from tests.emulation import Emulation
from tests.hf_oracle import save_and_convert

eng = pkg.engine
cv = pkg.convert

# Emulation (f16 form, float64 accumulation) against the HF float64 oracle, max |a - b| / max |b| per image, on the micro tower
# (2 layers, 17 tokens, 3 images).  Measured: image_embeds 3.2e-4 (QuickGELU) / 3.4e-4 (erf GELU), pooler_output 1.9e-4 / 2.3e-4,
# hidden_states[0] 2.0e-4, [1] 2.9e-4 / 3.0e-4, [2] 3.6e-4 / 3.7e-4: the f16 rounding of every GEMM operand and the reference's f16
# soft-max table, which the oracle does not have.
EMU_BOUND = 1e-3


@pytest.fixture(scope="module", params=["quick_gelu", "gelu_erf"])
def clip(request, tmp_path_factory):
    d = str(tmp_path_factory.mktemp(f"clip_{request.param}"))
    m = co.build_hf("micro", request.param)
    path = save_and_convert(m, d, "clip")
    imgs = gf.synthetic_images(3, 64, seed=3)
    return request.param, m, d, path, gf.read_gguf(path), imgs, co.hf_outputs(m, imgs)


def _distances(vf, imgs, o):
    emu = Emulation(vf, acc=np.float64, fp8=False)
    L = vf.num_hidden_layers
    x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
    d = {"image_embeds": fr.rel_dist(emu.forward(imgs), o["image_embeds"]).max(),
         "pooler_output": fr.rel_dist(emu.prelogits(x[L]), o["pooler_output"]).max()}
    d.update({f"hidden_states[{i}]": fr.rel_dist(x[i], o["hidden_states"][i]).max() for i in x})
    return d


def test_conversion_round_trip(clip):
    act, m, d, path, vf, _, _ = clip
    assert (vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.num_classes, vf.patch_size, vf.img_size) == (128, 2, 2, 96, 16, 64)
    assert np.float32(vf.eps) == np.float32(1e-5) and vf.pre_norm == 1 and vf.activation == act
    assert len(vf.tensors) == 4 + 12 * 2 + 4 + 2
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    D = 128
    qkv = np.asarray(vf.tensors["blocks.1.attn.qkv.weight"], np.float32)
    for i, x in enumerate("qkv"):
        assert np.array_equal(qkv[i * D:(i + 1) * D], sd[f"vision_model.encoder.layers.1.self_attn.{x}_proj.weight"])
    assert np.array_equal(vf.tensors["norm_pre.weight"], sd["vision_model.pre_layrnorm.weight"])
    assert np.array_equal(vf.tensors["norm.bias"], sd["vision_model.post_layernorm.bias"])
    assert np.array_equal(np.asarray(vf.tensors["head.weight"], np.float32), sd["visual_projection.weight"])
    assert not np.asarray(vf.tensors["head.bias"]).any() and not np.asarray(vf.tensors["patch_embed.proj.bias"]).any()
    assert np.array_equal(vf.tensors["pos_embed"].reshape(-1, D), sd["vision_model.embeddings.position_embedding.weight"])


def test_emulation_matches_the_hf_oracle(clip):
    act, _, _, _, vf, imgs, o = clip
    d = _distances(vf, imgs, o)
    print(act, {k: f"{v:.2e}" for k, v in d.items()})
    assert max(d.values()) <= EMU_BOUND, d


def test_a_broken_mapping_fails_the_oracle_check(clip):
    """q and k swapped, the pre-norm dropped and the other activation, each in the converted file: measured 0.47, 0.46 and 6e-3 on the
    image embeddings against <= 3.4e-4 for the right mapping.  The two activations differ by a few hundredths at most, so that bug shows
    by one order of magnitude rather than three."""
    act, _, _, _, vf, imgs, o = clip
    good = fr.rel_dist(Emulation(vf, acc=np.float64, fp8=False).forward(imgs), o["image_embeds"]).max()
    D = vf.hidden_size
    qk = copy.deepcopy(vf)
    for i in range(vf.num_hidden_layers):
        for p in ("weight", "bias"):
            w = np.array(qk.tensors[f"blocks.{i}.attn.qkv.{p}"])
            w[:2 * D] = np.concatenate([w[D:2 * D], w[:D]])
            qk.tensors[f"blocks.{i}.attn.qkv.{p}"] = w
    no_pre = copy.deepcopy(vf)
    no_pre.pre_norm = 0
    other = copy.deepcopy(vf)
    other.activation = "gelu_erf" if act == "quick_gelu" else "quick_gelu"
    bad = {n: fr.rel_dist(Emulation(b, acc=np.float64, fp8=False).forward(imgs), o["image_embeds"]).max()
           for n, b in (("qk", qk), ("no_pre", no_pre), ("activation", other))}
    print(act, f"right {good:.2e}", {k: f"{v:.2e}" for k, v in bad.items()})
    assert bad["qk"] > 300 * EMU_BOUND and bad["no_pre"] > 300 * EMU_BOUND
    assert bad["activation"] > 3 * EMU_BOUND and bad["activation"] > 10 * good


def test_timm_names_with_the_architecture_flags_give_the_same_file(clip, tmp_path):
    """The same weights under timm names (a CLIP-pretrained timm ViT), converted with --keep-norm-pre --activation --eps, give the file
    the CLIP converter writes, byte for byte; without the flags norm_pre is dropped as before."""
    act, m, d, path, vf, _, _ = clip
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    import json
    tsd, heads, activation, eps = cv.clip_to_timm(sd, json.load(open(os.path.join(d, "config.json"))))
    assert list(tsd)[:6] == ["cls_token", "pos_embed", "patch_embed.proj.weight", "patch_embed.proj.bias", "norm_pre.weight", "norm_pre.bias"]
    src = str(tmp_path / "timm.safetensors")
    cv.write_safetensors(src, tsd)
    out = str(tmp_path / "timm.gguf")
    cv.main([src, out, "--heads", str(heads), "--keep-norm-pre", "--activation", act, "--eps", "1e-5"])
    assert open(out, "rb").read() == open(path, "rb").read()
    plain = str(tmp_path / "plain.gguf")
    cv.main([src, plain, "--heads", str(heads), "--container", "gguf"])
    back = gf.read_gguf(plain)
    assert "norm_pre.weight" not in back.tensors and back.pre_norm == 0 and back.activation == "gelu_tanh"
    with pytest.raises(ValueError, match="needs --container gguf"):
        cv.main([src, str(tmp_path / "x.bin"), "--heads", str(heads), "--keep-norm-pre", "--container", "legacy"])


def test_reference_architecture_files_carry_no_new_keys(tmp_path):
    vf = gf.read(model_path("micro", "f16"))
    p = str(tmp_path / "m.gguf")
    gf.write_gguf(p, vf)
    raw = open(p, "rb").read()
    assert b"vit.pre_norm" not in raw and b"vit.activation" not in raw
    back = gf.read_gguf(p)
    assert (back.pre_norm, back.activation, np.float32(back.eps)) == (0, "gelu_tanh", np.float32(1e-6))


def test_clip_converter_refusals(clip, tmp_path):
    _, m, d, _, _, _, _ = clip
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    act = clip[0]
    cfg = {"hidden_act": co.HF_ACT[act], "num_attention_heads": 2, "layer_norm_eps": 1e-5}
    out = str(tmp_path / "x.gguf")
    with pytest.raises(ValueError, match="hidden_act 'gelu_pytorch_tanh' is not supported"):
        cv.clip_to_model_file(sd, dict(cfg, hidden_act="gelu_pytorch_tanh"), out)
    with pytest.raises(ValueError, match="head dim 32 is not supported"):
        cv.clip_to_model_file(sd, dict(cfg, num_attention_heads=4), out)
    narrow = dict(sd)
    narrow["vision_model.encoder.layers.0.mlp.fc1.weight"] = sd["vision_model.encoder.layers.0.mlp.fc1.weight"][:3 * 128]
    with pytest.raises(ValueError, match="intermediate size 384 is not supported"):
        cv.clip_to_model_file(narrow, cfg, out)
    with pytest.raises(ValueError, match="needs --container gguf"):
        cv.clip_to_model_file(sd, cfg, out, container="legacy")
    # the CLI: a full CLIPModel's config nests the vision tower's fields; text_model.* and friends are ignored
    full = dict(sd, **{"text_model.embeddings.token_embedding.weight": np.zeros((8, 4), np.float32), "logit_scale": np.zeros((), np.float32),
                       "text_projection.weight": np.zeros((4, 4), np.float32)})
    src = str(tmp_path / "full.safetensors")
    cv.write_safetensors(src, full)
    cfgp = co.write_config(str(tmp_path), vision_config=cfg, text_config={"hidden_act": "relu"})
    cv.main([src, out, "--hf-config", cfgp])
    assert open(out, "rb").read() == open(os.path.join(d, "clip.gguf"), "rb").read()
    with pytest.raises(SystemExit, match="needs --hf-config"):
        cv.main([src, out])
    with pytest.raises(ValueError, match="needs --container gguf"):
        cv.main([src, out, "--hf-config", cfgp, "--container", "legacy"])


def test_engine_refusals_need_no_gpu(clip, tmp_path):
    """Checked before the device is touched, so they are testable anywhere: a bad vitb200_arch field, pre_norm = 1 without the norm_pre
    tensors, and a GGUF file whose vit.activation is unknown."""
    _, _, _, path, vf, _, _ = clip
    with pytest.raises(eng.VitB200Error, match="vitb200_arch.pre_norm = 2 out of range"):
        _create_arch(vf, 2, 0)
    with pytest.raises(eng.VitB200Error, match="vitb200_arch.activation = 3 out of range"):
        _create_arch(vf, 1, 3)
    relu = copy.deepcopy(vf)
    relu.activation = "relu"
    with pytest.raises(eng.VitB200Error, match="vitb200_arch.activation = -1 out of range"):
        eng.vit_model_from_tensors(relu, 0, 2)
    missing = copy.deepcopy(vf)
    del missing.tensors["norm_pre.bias"]
    with pytest.raises(eng.VitB200Error, match="pre_norm = 1 needs the tensors 'norm_pre.weight' and 'norm_pre.bias'"):
        eng.vit_model_from_tensors(missing, 0, 2)
    raw = open(path, "rb").read()
    key = b"vit.activation"
    i = raw.index(key) + len(key) + 4       # past the key and the value type: {u64 length, bytes}
    n = int.from_bytes(raw[i:i + 8], "little")
    p = tmp_path / "relu.gguf"
    p.write_bytes(raw[:i] + (4).to_bytes(8, "little") + b"relu" + raw[i + 8 + n:])
    with pytest.raises(eng.VitB200Error, match="unknown vit.activation 'relu'"):
        eng.vit_model_load(str(p))


def _create_arch(vf, pre_norm, activation):
    """vitb200_create_arch with explicit fields (vit_model_from_tensors maps names, so it cannot pass an out-of-range index)."""
    import ctypes as C
    L = eng.lib()
    entries = [(n.encode(), np.ascontiguousarray(a, np.float16 if vf.tensor_ftype[n] == 1 else np.float32), vf.tensor_ftype[n])
               for n, a in vf.tensors.items()]
    ts = (eng.Tensor * len(entries))()
    for t, (nm, a, ft) in zip(ts, entries):
        t.name, t.data, t.type, t.n_dims = nm, a.ctypes.data, ft, a.ndim
        for i, dim in enumerate(reversed(a.shape)):
            t.ne[i] = dim
    hp = eng.Hparams(vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.num_classes, vf.patch_size, vf.img_size, 1, vf.eps)
    h = C.c_void_p()
    eng._check(L.vitb200_create_arch(C.byref(hp), C.byref(eng.Arch(pre_norm, activation)), ts, len(entries), 0, 2, 1, 0, C.byref(h)),
               "vitb200_create_arch")


def test_gguf_parser_fuzzed_with_the_architecture_keys(clip, tmp_path):
    """tests/cpp/gguf_fuzz.cpp under ASan / UBSan with a CLIP file as its GGUF seed: truncations and byte flips of a file that carries
    vit.pre_norm and vit.activation (whose string value the parser maps and may reject)."""
    act, _, _, path, _, _, _ = clip
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("no g++")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "gguf_fuzz")
    r = subprocess.run([gxx, "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-I", os.path.join(root, "vit.cpp_b200", "csrc"), os.path.join(root, "tests", "cpp", "gguf_fuzz.cpp"), "-o", exe],
                       capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr.lower():
        pytest.skip("sanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe, path, model_path("micro", "f16")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert r.stdout.count("rejected") == 2   # both parsers ran
