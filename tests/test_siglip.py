"""SigLIP on the CPU: the Hugging Face converter for SiglipVisionModel, the vision tower of SiglipModel and SiglipForImageClassification,
the GGUF values vit.pool "map" / "mean" and vit.activation "gelu_pytorch_tanh", the emulation against an independent float64
oracle (transformers' SigLIP classes), and the refusals that need no GPU."""
import copy
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.util import pkg, gf, model_path
from tests import siglip_oracle as so
from tests import fp8_reference as fr
from tests.emulation import Emulation
from tests.hf_oracle import save_and_convert

eng = pkg.engine
cv = pkg.convert

# Emulation (f16 form, float64 accumulation) against the HF float64 oracle, max |a - b| / max |b| per image, on the micro towers (2 layers,
# 16 tokens, 3 images).  Measured: 2.0e-4 .. 6.6e-4 on the logits, prelogits and hidden_states[0, 1, 2] of both classes: the f16 rounding
# of every GEMM operand and the reference's f16 soft-max table, which the oracle does not have.
EMU_BOUND = 1.5e-3
CLASSES = [False, True]
IDS = ["SiglipVisionModel", "SiglipForImageClassification"]


@pytest.fixture(scope="module", params=CLASSES, ids=IDS)
def sig(request, tmp_path_factory):
    classifier = request.param
    d = str(tmp_path_factory.mktemp(f"siglip_{classifier}"))
    m = so.build_hf("micro", classifier)
    path = save_and_convert(m, d, "siglip")
    imgs = gf.synthetic_images(3, so.image_size("micro"), seed=3)
    return classifier, m, d, path, gf.read_gguf(path), imgs, so.hf_outputs(m, imgs)


def _distances(vf, imgs, o, emu=None):
    emu = emu or Emulation(vf, acc=np.float64, fp8=False)
    L = vf.num_hidden_layers
    x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
    d = {"logits": fr.rel_dist(emu.forward(imgs), o["logits"]).max(), "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["prelogits"]).max()}
    d.update({f"hidden_states[{i}]": fr.rel_dist(x[i], o["hidden_states"][i]).max() for i in x})
    return d


def test_conversion_round_trip(sig):
    classifier, m, _, _, vf, _, _ = sig
    D, L = 128, 2
    assert (vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.patch_size, vf.img_size) == (D, L, 2, 16, 64)
    assert vf.num_classes == (so.NUM_LABELS if classifier else D)
    assert (vf.pool, vf.activation, vf.pre_norm, vf.layer_scale, vf.reg_tokens) == ("mean" if classifier else "map", "gelu_pytorch_tanh", 0, 0, 0)
    assert np.float32(vf.eps) == np.float32(1e-6) and vf.n_tokens == 16
    assert len(vf.tensors) == 12 * L + (7 if classifier else 20)
    assert "cls_token" not in vf.tensors and vf.tensors["pos_embed"].shape == (1, 16, D)
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    h = "vision_model.encoder.layers.1."
    qkv = np.asarray(vf.tensors["blocks.1.attn.qkv.weight"], np.float32)
    for i, x in enumerate("qkv"):
        assert np.array_equal(qkv[i * D:(i + 1) * D], sd[f"{h}self_attn.{x}_proj.weight"])
    assert np.array_equal(np.asarray(vf.tensors["blocks.1.mlp.fc2.weight"], np.float32), sd[h + "mlp.fc2.weight"])
    assert np.array_equal(vf.tensors["norm.bias"], sd["vision_model.post_layernorm.bias"])
    assert np.array_equal(vf.tensors["pos_embed"].reshape(16, D), sd["vision_model.embeddings.position_embedding.weight"])
    assert np.array_equal(vf.tensors["patch_embed.proj.bias"].reshape(D), sd["vision_model.embeddings.patch_embedding.bias"])
    if classifier:
        assert np.array_equal(np.asarray(vf.tensors["head.weight"], np.float32), sd["classifier.weight"])
        assert not any(k.startswith("attn_pool.") for k in vf.tensors)
        return
    assert np.array_equal(np.asarray(vf.tensors["head.weight"], np.float32), np.eye(D)) and not np.asarray(vf.tensors["head.bias"]).any()
    w, b = sd["vision_model.head.attention.in_proj_weight"], sd["vision_model.head.attention.in_proj_bias"]
    assert np.array_equal(np.asarray(vf.tensors["attn_pool.q.weight"], np.float32), w[:D])
    assert np.array_equal(np.asarray(vf.tensors["attn_pool.kv.weight"], np.float32), w[D:])     # rows k then v
    assert np.array_equal(vf.tensors["attn_pool.kv.bias"], b[D:])
    assert vf.tensors["attn_pool.latent"].dtype == np.float32
    assert np.array_equal(vf.tensors["attn_pool.latent"], sd["vision_model.head.probe"])
    assert np.array_equal(np.asarray(vf.tensors["attn_pool.proj.weight"], np.float32), sd["vision_model.head.attention.out_proj.weight"])
    assert np.array_equal(vf.tensors["attn_pool.norm.weight"], sd["vision_model.head.layernorm.weight"])
    assert np.array_equal(np.asarray(vf.tensors["attn_pool.mlp.fc1.weight"], np.float32), sd["vision_model.head.mlp.fc1.weight"])


def test_siglip_model_vision_tower_converts_like_the_vision_model(sig, tmp_path):
    """A full SiglipModel state dict (text tower, logit_scale, logit_bias) with the same vision weights converts to the same bytes."""
    classifier, m, d, path, _, _, _ = sig
    if classifier:
        pytest.skip("the SiglipModel case is the vision tower without a classifier")
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    full = dict(sd, **{"text_model.embeddings.token_embedding.weight": np.zeros((8, 4), np.float32),
                       "logit_scale": np.zeros((1,), np.float32), "logit_bias": np.zeros((1,), np.float32)})
    src = str(tmp_path / "full.safetensors")
    cv.write_safetensors(src, full)
    cfg = json.load(open(os.path.join(d, "config.json")))
    cfgp = str(tmp_path / "config.json")
    json.dump({"model_type": "siglip", "vision_config": cfg, "text_config": {"hidden_act": "gelu_pytorch_tanh"}}, open(cfgp, "w"))
    out = str(tmp_path / "full.gguf")
    cv.main([src, out, "--hf-config", cfgp])
    assert open(out, "rb").read() == open(path, "rb").read()


def test_emulation_matches_the_hf_oracle(sig):
    classifier, _, _, _, vf, imgs, o = sig
    d = _distances(vf, imgs, o)
    print(IDS[classifier], {k: f"{v:.2e}" for k, v in d.items()})
    assert max(d.values()) <= EMU_BOUND, d


class _PreLnPool(Emulation):
    """Pools the residual stream without the final LayerNorm."""

    def prelogits(self, x, norm=True):
        y = np.asarray(x, np.float32)
        return self.map_head(y) if self.pool == "map" else y.astype(np.float64).mean(axis=1).astype(np.float32)


class _NoMlpResidual(Emulation):
    """The head's MLP output without the residual h."""

    def map_head(self, y):
        return self.head_mlp(self.pool_attention(y))


def test_a_broken_mapping_fails_the_oracle_check(sig):
    """k and v swapped, pooling over the pre-LN rows, the head's MLP residual dropped, positions offset by one row (the class-token bug):
    each lands far outside the bound the right mapping meets."""
    classifier, _, _, _, vf, imgs, o = sig
    D = vf.hidden_size
    bad = {}
    if not classifier:
        swapped = copy.deepcopy(vf)
        for n in ("attn_pool.kv.weight", "attn_pool.kv.bias"):
            a = swapped.tensors[n]
            swapped.tensors[n] = np.concatenate([a[D:], a[:D]])
        bad["k and v swapped"] = _distances(swapped, imgs, o)
        bad["MLP residual dropped"] = _distances(vf, imgs, o, _NoMlpResidual(vf, acc=np.float64, fp8=False))
    bad["pooled over pre-LN rows"] = _distances(vf, imgs, o, _PreLnPool(vf, acc=np.float64, fp8=False))
    shifted = copy.deepcopy(vf)
    pos = shifted.tensors["pos_embed"].reshape(-1, D)
    shifted.tensors["pos_embed"] = np.concatenate([pos[1:], pos[:1]]).reshape(1, -1, D)   # patch p takes position row p + 1
    bad["positions offset by one row"] = _distances(shifted, imgs, o)
    worst = {k: max(v.values()) for k, v in bad.items()}
    print(IDS[classifier], {k: f"{v:.2e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v > 10 * EMU_BOUND, (k, v)


def test_reference_clip_and_dinov2_files_carry_no_new_keys(tmp_path):
    """No new value or tensor in a reference, CLIP or DINOv2 file, and the writer reproduces each of them byte for byte."""
    from tests import clip_oracle as co
    from tests import dinov2_oracle as do
    vf = gf.read(model_path("micro", "f16"))
    p = str(tmp_path / "m.gguf")
    gf.write_gguf(p, vf)
    clip = save_and_convert(co.build_hf("micro"), str(tmp_path / "clip"), "clip")
    dino = save_and_convert(do.build_hf("micro_reg", True), str(tmp_path / "dino"), "dinov2", do.convert_size("micro_reg"))
    for f in (p, clip, dino):
        raw = open(f, "rb").read()
        assert b"gelu_pytorch_tanh" not in raw and b"attn_pool" not in raw
        back = gf.read_gguf(f)
        assert back.pool in ("token", "cls_patch_mean") and back.activation != "gelu_pytorch_tanh"
        again = str(tmp_path / "again.gguf")
        gf.write_gguf(again, back)
        assert open(again, "rb").read() == raw


def test_siglip_converter_refusals(sig, tmp_path):
    classifier, m, d, _, _, _, _ = sig
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    cfg = {"hidden_act": "gelu_pytorch_tanh", "num_attention_heads": 2, "layer_norm_eps": 1e-6, "intermediate_size": 512}
    out = str(tmp_path / "x.gguf")
    cases = [(dict(cfg, hidden_act="gelu"), "hidden_act 'gelu' is not supported"),
             (dict(cfg, num_attention_heads=4), "head dim 32 is not supported"),
             # So400m: hidden 1152, 16 heads (head dim 72), MLP 4304
             (dict(cfg, num_attention_heads=16, intermediate_size=4304), "head dim 8 is not supported"),
             (dict(cfg, intermediate_size=4304), "intermediate_size 4304 is not supported")]
    if not classifier:
        cases.append((dict(cfg, vision_use_head=False), "vision_use_head = false is not supported"))
    for bad, msg in cases:
        with pytest.raises(ValueError, match=msg):
            cv.siglip_to_model_file(sd, bad, out)
    with pytest.raises(ValueError, match="needs --container gguf"):
        cv.siglip_to_model_file(sd, cfg, out, container="legacy")
    with pytest.raises(SystemExit, match="needs --hf-config"):
        cv.main([os.path.join(d, "model.safetensors"), out])
    assert cv.is_hf_siglip(sd)


def _create(vf, arch, head_tokens=1, edit=None):
    """vitb200_create_arch with explicit fields, on no GPU: every refusal below comes before the device check."""
    entries = [(n, np.ascontiguousarray(a, np.float16 if vf.tensor_ftype[n] == 1 else np.float32), vf.tensor_ftype[n])
               for n, a in vf.tensors.items()]
    if edit:
        entries = edit(entries)
    ts = (eng.Tensor * len(entries))()
    for t, (nm, a, ft) in zip(ts, entries):
        t.name, t.data, t.type, t.n_dims = nm.encode(), a.ctypes.data, ft, a.ndim
        for i, dim in enumerate(reversed(a.shape)):
            t.ne[i] = dim
    hp = eng.Hparams(vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.num_classes, vf.patch_size, vf.img_size, 1, vf.eps)
    h = C.c_void_p()
    eng._check(eng.lib().vitb200_create_arch(C.byref(hp), C.byref(arch), ts, len(entries), 0, 2, head_tokens, 0, C.byref(h)),
               "vitb200_create_arch")


def test_engine_refusals_need_no_gpu(sig, tmp_path):
    classifier, _, _, path, vf, _, _ = sig
    pool = 3 if classifier else 2
    ok = lambda **kw: eng.Arch(**dict(dict(pre_norm=0, activation=3, layer_scale=0, reg_tokens=0, pool=pool), **kw))
    drop = lambda name: (lambda es: [e for e in es if e[0] != name])
    add_cls = lambda es: es + [("cls_token", np.zeros((1, 1, vf.hidden_size), np.float32), 0)]
    cases = [(ok(pool=4), "vitb200_arch.pool = 4 out of range"), (ok(activation=4), "vitb200_arch.activation = 4 out of range"),
             (ok(reg_tokens=4), f"vitb200_arch.pool = {pool} needs reg_tokens = 0"),
             (ok(pool=1), "vitb200_arch.activation = 3 out of range for pool 1"),
             (ok(pool=0), "vitb200_arch.activation = 3 out of range for pool 0")]
    for arch, msg in cases:
        with pytest.raises(eng.VitB200Error, match=msg):
            _create(vf, arch)
    with pytest.raises(eng.VitB200Error, match=f"pool = {pool} needs head_tokens = 1"):
        _create(vf, ok(), head_tokens=2)
    with pytest.raises(eng.VitB200Error, match=f"vitb200_arch.pool = {pool} out of range for a model with a class token"):
        _create(vf, ok(), edit=add_cls)
    longer = lambda es: [(n, np.concatenate([a, a[:, :1]], axis=1) if n == "pos_embed" else a, ft) for n, a, ft in es]
    with pytest.raises(eng.VitB200Error, match=f"pool = {pool} needs 'pos_embed' with the 16 patch rows only .* got 17 rows"):
        _create(vf, ok(), edit=longer)
    wide = lambda es: [(n, np.concatenate([a, a], axis=1) if n == "head.weight" else a, ft) for n, a, ft in es]
    with pytest.raises(eng.VitB200Error, match=f"pool = {pool} needs 'head.weight' with K = 128"):
        _create(vf, ok(), edit=wide)
    if not classifier:
        for name in ("attn_pool.latent", "attn_pool.kv.bias", "attn_pool.mlp.fc2.weight"):
            with pytest.raises(eng.VitB200Error, match=f"pool = 2 needs the attention-pooling head's tensor '{name}'"):
                _create(vf, ok(), edit=drop(name))
    big = copy.deepcopy(vf)
    big.img_size = 16 * 30                                  # 900 patch rows > 896 tokens
    big.tensors["pos_embed"] = np.zeros((1, 900, vf.hidden_size), np.float32)
    with pytest.raises(eng.VitB200Error, match="900 tokens not supported"):
        _create(big, ok())
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(eng.VitB200Error, match="no CPU fallback"):
            _create(vf, ok())                               # everything else is in order: the device check is next
    # the model file: its tensor count (12 L + 20 or 12 L + 7) and its vit.pool string
    short = copy.deepcopy(vf)
    del short.tensors["blocks.1.norm1.bias"]
    p = str(tmp_path / "short.gguf")
    gf.write_gguf(p, short)
    with pytest.raises(eng.VitB200Error, match=f"model file has {12 * 2 + (6 if classifier else 19)} tensors, but "
                                                f"{12 * 2 + (7 if classifier else 20)} tensors were expected"):
        eng.vit_model_load(p)
    raw = open(path, "rb").read()
    key = b"vit.pool"
    i = raw.index(key) + len(key) + 4
    n = int.from_bytes(raw[i:i + 8], "little")
    q = tmp_path / "avg.gguf"
    q.write_bytes(raw[:i] + (3).to_bytes(8, "little") + b"avg" + raw[i + 8 + n:])
    with pytest.raises(eng.VitB200Error, match=r"unknown vit.pool 'avg' \(token, cls_patch_mean, map or mean\)"):
        eng.vit_model_load(str(q))


def test_arch_struct_layout_is_unchanged():
    assert C.sizeof(eng.Arch) == 20
    assert [(n, getattr(eng.Arch, n).offset) for n, _ in eng.Arch._fields_] == [
        ("pre_norm", 0), ("activation", 4), ("layer_scale", 8), ("reg_tokens", 12), ("pool", 16)]
    assert gf.POOLS == ("token", "cls_patch_mean", "map", "mean")
    assert gf.ACTIVATIONS == ("gelu_tanh", "gelu_erf", "quick_gelu", "gelu_pytorch_tanh")


def test_gguf_parser_fuzzed_with_a_siglip_file(sig, tmp_path):
    """tests/cpp/gguf_fuzz.cpp under ASan / UBSan with a SigLIP file (vit.pool "map", vit.activation "gelu_pytorch_tanh", the
    attention-pooling head's tensors) as its GGUF seed."""
    classifier, _, _, path, _, _, _ = sig
    if classifier:
        pytest.skip("one seed carrying every new value is enough")
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
    raw = open(path, "rb").read()
    assert b"gelu_pytorch_tanh" in raw and b"attn_pool.latent" in raw and b"map" in raw
    r = subprocess.run([exe, path, model_path("micro", "f16")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert r.stdout.count("rejected") == 2
