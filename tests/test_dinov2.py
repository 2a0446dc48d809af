"""DINOv2 on the CPU: the Hugging Face converter for all four classes, the position-grid resampling, the GGUF keys vit.layer_scale /
vit.reg_tokens / vit.pool, the emulation against an independent float64 oracle (transformers' DINOv2 classes), and the
refusals that need no GPU."""
import copy
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.util import pkg, gf, model_path
from tests import dinov2_oracle as do
from tests import fp8_reference as fr
from tests.emulation import Emulation
from tests.hf_oracle import save_and_convert

eng = pkg.engine
cv = pkg.convert

# Emulation (f16 form, float64 accumulation) against the HF float64 oracle, max |a - b| / max |b| per image, on the micro models
# (2 layers, 17 or 21 tokens, 3 images).  Measured: 1.1e-4 .. 6.4e-4 on the logits, prelogits and hidden_states[0, 1, 2] of the four
# classes: the f16 rounding of every GEMM operand and the reference's f16 soft-max table, which the oracle does not have.
EMU_BOUND = 1.5e-3
CLASSES = [("micro", True), ("micro", False), ("micro_reg", True), ("micro_reg", False)]
IDS = ["Dinov2ForImageClassification", "Dinov2Model", "Dinov2WithRegistersForImageClassification", "Dinov2WithRegistersModel"]


@pytest.fixture(scope="module", params=CLASSES, ids=IDS)
def dino(request, tmp_path_factory):
    geo, classifier = request.param
    d = str(tmp_path_factory.mktemp(f"dino_{geo}_{classifier}"))
    m = do.build_hf(geo, classifier)
    path = save_and_convert(m, d, "dinov2", do.convert_size(geo))
    imgs = gf.synthetic_images(3, do.image_size(geo), seed=3)
    return geo, classifier, m, d, path, gf.read_gguf(path), imgs, do.hf_outputs(m, imgs)


def _distances(vf, imgs, o, emu=None):
    emu = emu or Emulation(vf, acc=np.float64, fp8=False)
    L = vf.num_hidden_layers
    x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
    d = {"logits": fr.rel_dist(emu.forward(imgs), o["logits"]).max(), "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["prelogits"]).max()}
    d.update({f"hidden_states[{i}]": fr.rel_dist(x[i], o["hidden_states"][i]).max() for i in x})
    return d


def test_conversion_round_trip(dino):
    geo, classifier, m, _, _, vf, _, _ = dino
    D, R, L = 128, do.GEOMETRIES[geo][5], 2
    assert (vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.patch_size, vf.img_size) == (D, L, 2, 14, 56)
    assert vf.num_classes == (do.NUM_LABELS if classifier else D)
    assert (vf.layer_scale, vf.reg_tokens, vf.pool, vf.activation, vf.pre_norm) == (1, R, "cls_patch_mean" if classifier else "token", "gelu_erf", 0)
    assert np.float32(vf.eps) == np.float32(1e-6) and vf.n_tokens == 16 + 1 + R
    assert len(vf.tensors) == 4 + 12 * L + 4 + 2 * L + (R > 0)
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    pre = {"micro": "dinov2.", "micro_reg": "dinov2_with_registers."}[geo] if classifier else ""
    h = f"{pre}encoder.layer.1."
    qkv = np.asarray(vf.tensors["blocks.1.attn.qkv.weight"], np.float32)
    for i, x in enumerate(("query", "key", "value")):
        assert np.array_equal(qkv[i * D:(i + 1) * D], sd[f"{h}attention.attention.{x}.weight"])
    assert np.array_equal(vf.tensors["blocks.1.ls1.gamma"], sd[h + "layer_scale1.lambda1"])
    assert np.array_equal(vf.tensors["blocks.1.ls2.gamma"], sd[h + "layer_scale2.lambda1"])
    assert np.array_equal(np.asarray(vf.tensors["blocks.1.attn.proj.weight"], np.float32), sd[h + "attention.output.dense.weight"])
    assert np.array_equal(vf.tensors["norm.bias"], sd[pre + "layernorm.bias"])
    pos = vf.tensors["pos_embed"].reshape(-1, D)
    assert np.array_equal(pos[0], sd[pre + "embeddings.position_embeddings"].reshape(-1, D)[0]) and not pos[1:1 + R].any()
    if R:
        assert vf.tensors["reg_token"].dtype == np.float32
        assert np.array_equal(vf.tensors["reg_token"].reshape(R, D), sd[pre + "embeddings.register_tokens"].reshape(R, D))
    if classifier:
        assert np.array_equal(np.asarray(vf.tensors["head.weight"], np.float32), sd["classifier.weight"])
    else:
        assert np.array_equal(np.asarray(vf.tensors["head.weight"], np.float32), np.eye(D)) and not np.asarray(vf.tensors["head.bias"]).any()
    assert not any("mask_token" in k for k in vf.tensors)


def test_resampled_pos_embed_is_hf_interpolate_pos_encoding(dino):
    """The converter's resampled patch rows are what HF's interpolate_pos_encoding computes at run time for the converted size."""
    import torch
    geo, _, m, _, _, vf, _, _ = dino
    D, R, S = 128, do.GEOMETRIES[geo][5], do.image_size(geo)
    emb = do.backbone(m).embeddings
    with torch.no_grad():
        want = emb.interpolate_pos_encoding(torch.zeros(1, 17, D), S, S).numpy().reshape(-1, D)
    got = vf.tensors["pos_embed"].reshape(-1, D)
    assert got.shape[0] == 17 + R
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1 + R:], want[1:])


def test_emulation_matches_the_hf_oracle(dino):
    geo, classifier, _, _, _, vf, imgs, o = dino
    d = _distances(vf, imgs, o)
    print(geo, classifier, {k: f"{v:.2e}" for k, v in d.items()})
    assert max(d.values()) <= EMU_BOUND, d


def test_a_broken_mapping_fails_the_oracle_check(dino):
    """gamma dropped, registers given position rows, registers counted in the patch mean, the class token mean-pooled with the patches:
    each lands far outside the bound the right mapping meets."""
    geo, classifier, _, _, _, vf, imgs, o = dino
    R = vf.reg_tokens
    bad = {}
    no_gamma = copy.deepcopy(vf)
    no_gamma.layer_scale = 0
    bad["gamma dropped"] = _distances(no_gamma, imgs, o)
    if R:
        shifted = copy.deepcopy(vf)
        pos = shifted.tensors["pos_embed"].reshape(-1, vf.hidden_size).copy()
        pos[1:1 + R] = pos[1 + R:1 + 2 * R]                                 # registers given (patch) position rows
        shifted.tensors["pos_embed"] = pos.reshape(1, -1, vf.hidden_size)
        bad["register position rows"] = _distances(shifted, imgs, o)
    if classifier:
        class RegsInMean(Emulation):
            def prelogits(self, x, norm=True):
                y = rs_ln(self, x)
                return np.concatenate([y[:, 0], y[:, 1:].mean(axis=1)], axis=1)

        class ClsInMean(Emulation):
            def prelogits(self, x, norm=True):
                y = rs_ln(self, x)
                return np.concatenate([y[:, 0], np.concatenate([y[:, :1], y[:, 1 + self.R:]], axis=1).mean(axis=1)], axis=1)

        if R:
            bad["registers in the mean"] = _distances(vf, imgs, o, RegsInMean(vf, acc=np.float64, fp8=False))
        bad["cls mean-pooled"] = _distances(vf, imgs, o, ClsInMean(vf, acc=np.float64, fp8=False))
    worst = {k: max(v.values()) for k, v in bad.items()}
    print(geo, classifier, {k: f"{v:.2e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v > 10 * EMU_BOUND, (k, v)


def rs_ln(emu, x):
    from oracle import restatement as rs
    x = np.asarray(x, np.float32)
    B, N, D = x.shape
    return rs.layernorm(x.reshape(-1, D), emu.norm_w, emu.norm_b, emu.eps).reshape(B, N, D)


def test_reference_and_clip_files_carry_no_new_keys(tmp_path):
    from tests import clip_oracle as co
    vf = gf.read(model_path("micro", "f16"))
    p = str(tmp_path / "m.gguf")
    gf.write_gguf(p, vf)
    clip = save_and_convert(co.build_hf("micro"), str(tmp_path / "clip"), "clip")
    for f in (p, clip):
        raw = open(f, "rb").read()
        assert b"vit.layer_scale" not in raw and b"vit.reg_tokens" not in raw and b"vit.pool" not in raw
        back = gf.read_gguf(f)
        assert (back.layer_scale, back.reg_tokens, back.pool) == (0, 0, "token")


def test_dinov2_converter_refusals(dino, tmp_path):
    _, _, m, d, path, _, _, _ = dino
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    cfg = {"hidden_act": "gelu", "num_attention_heads": 2, "layer_norm_eps": 1e-6}
    out = str(tmp_path / "x.gguf")
    for bad, msg in ((dict(cfg, use_swiglu_ffn=True), "use_swiglu_ffn"), (dict(cfg, num_attention_heads=4), "head dim 32 is not supported"),
                     (dict(cfg, mlp_ratio=2), "mlp_ratio 2 is not supported"), (dict(cfg, qkv_bias=False), "qkv_bias false is not supported"),
                     (dict(cfg, hidden_act="relu"), "hidden_act 'relu' is not supported")):
        with pytest.raises(ValueError, match=msg):
            cv.dinov2_to_model_file(sd, bad, out)
    with pytest.raises(ValueError, match="needs --container gguf"):
        cv.dinov2_to_model_file(sd, cfg, out, container="legacy")
    with pytest.raises(SystemExit, match="needs --hf-config"):
        cv.main([os.path.join(d, "model.safetensors"), out])
    with pytest.raises(ValueError, match="not a multiple of the patch size"):
        cv.dinov2_to_model_file(sd, cfg, out, img_size=60)


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


def test_engine_refusals_need_no_gpu(dino, tmp_path):
    geo, classifier, _, _, path, vf, _, _ = dino
    R, pool = vf.reg_tokens, int(classifier)
    ok = lambda **kw: eng.Arch(**dict(dict(pre_norm=0, activation=1, layer_scale=1, reg_tokens=R, pool=pool), **kw))
    for arch, msg in ((ok(layer_scale=2), "vitb200_arch.layer_scale = 2 out of range"), (ok(reg_tokens=17), "vitb200_arch.reg_tokens = 17 out of range"),
                      (ok(reg_tokens=-1), "vitb200_arch.reg_tokens = -1 out of range"), (ok(pool=2), "vitb200_arch.pool = 2 out of range"),
                      (ok(pool=1 - pool), "needs 'head.weight' with K = ")):
        with pytest.raises(eng.VitB200Error, match=msg):
            _create(vf, arch)
    drop = lambda name: (lambda es: [e for e in es if e[0] != name])
    with pytest.raises(eng.VitB200Error, match=r"layer_scale = 1 needs the tensor 'blocks.1.ls2.gamma'"):
        _create(vf, ok(), edit=drop("blocks.1.ls2.gamma"))
    if R:
        with pytest.raises(eng.VitB200Error, match="reg_tokens = 4 needs the tensor 'reg_token'"):
            _create(vf, ok(), edit=drop("reg_token"))
    if classifier:
        with pytest.raises(eng.VitB200Error, match="pool = 1 needs head_tokens = 1"):
            _create(vf, ok(), head_tokens=2)
    big = copy.deepcopy(vf)
    big.img_size = 14 * 30                                  # 900 patches + 1 + R > 896 tokens
    with pytest.raises(eng.VitB200Error, match=f"{901 + R} tokens not supported"):
        _create(big, ok())
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(eng.VitB200Error, match="no CPU fallback"):
            _create(vf, ok())                               # everything else is in order: the device check is next
    raw = open(path, "rb").read()
    if classifier:
        key = b"vit.pool"
        i = raw.index(key) + len(key) + 4
        n = int.from_bytes(raw[i:i + 8], "little")
        p = tmp_path / "avg.gguf"
        p.write_bytes(raw[:i] + (3).to_bytes(8, "little") + b"avg" + raw[i + 8 + n:])
        with pytest.raises(eng.VitB200Error, match="unknown vit.pool 'avg'"):
            eng.vit_model_load(str(p))


def test_arch_struct_layout():
    """vitb200_arch through ctypes: five int32 fields in the header's order; the positional two-field form still builds a CLIP tower."""
    assert C.sizeof(eng.Arch) == 20
    assert [(n, getattr(eng.Arch, n).offset) for n, _ in eng.Arch._fields_] == [
        ("pre_norm", 0), ("activation", 4), ("layer_scale", 8), ("reg_tokens", 12), ("pool", 16)]
    a = eng.Arch(1, 2)
    assert (a.pre_norm, a.activation, a.layer_scale, a.reg_tokens, a.pool) == (1, 2, 0, 0, 0)
    hdr = open(eng.HEADER_PATH).read()
    body = hdr[hdr.index("typedef struct vitb200_arch"):hdr.index("} vitb200_arch;")]
    import re
    assert re.findall(r"int32_t (\w+);", body) == [n for n, _ in eng.Arch._fields_]


def test_gguf_parser_fuzzed_with_the_dinov2_keys(dino, tmp_path):
    """tests/cpp/gguf_fuzz.cpp under ASan / UBSan with a DINOv2 file (vit.layer_scale, vit.reg_tokens, vit.pool) as its GGUF seed."""
    geo, classifier, _, _, path, _, _, _ = dino
    if not (geo == "micro_reg" and classifier):
        pytest.skip("one seed carrying every key is enough")
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
    assert b"vit.layer_scale" in raw and b"vit.reg_tokens" in raw and b"cls_patch_mean" in raw
    r = subprocess.run([exe, path, model_path("micro", "f16")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert r.stdout.count("rejected") == 2
