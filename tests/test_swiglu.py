"""SwiGLU MLPs (DINOv2 ViT-g, vitb200_arch.activation = 4) on the CPU: the Hugging Face converter for all four DINOv2 classes with
use_swiglu_ffn, the GGUF key vit.activation = "swiglu", the emulation against the float64 HF oracle, and the refusals that need no GPU."""
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

# Emulation (f16 form, float64 accumulation) against the HF float64 oracle, max |a - b| / max |b| per image, on the micro SwiGLU models
# (2 layers, F = 344, 17 or 21 tokens, 3 images).  Measured: 1.5e-4 .. 4.2e-4 on the logits, prelogits and hidden_states[0, 1, 2] of the
# four classes: the f16 rounding of every GEMM operand (h included) and the reference's f16 soft-max table, which the oracle does not have.
EMU_BOUND = 1e-3
CLASSES = [("micro", True), ("micro", False), ("micro_reg", True), ("micro_reg", False)]
IDS = ["Dinov2ForImageClassification", "Dinov2Model", "Dinov2WithRegistersForImageClassification", "Dinov2WithRegistersModel"]
D, F = 128, 344


@pytest.fixture(scope="module", params=CLASSES, ids=IDS)
def dino(request, tmp_path_factory):
    geo, classifier = request.param
    d = str(tmp_path_factory.mktemp(f"swiglu_{geo}_{classifier}"))
    m = do.build_hf(geo, classifier, swiglu=True)
    path = save_and_convert(m, d, "dinov2", do.convert_size(geo))
    imgs = gf.synthetic_images(3, do.image_size(geo), seed=3)
    return geo, classifier, m, d, path, gf.read_gguf(path), imgs, do.hf_outputs(m, imgs)


def _distances(vf, imgs, o):
    emu = Emulation(vf, acc=np.float64, fp8=False)
    L = vf.num_hidden_layers
    x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
    d = {"logits": fr.rel_dist(emu.forward(imgs), o["logits"]).max(), "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["prelogits"]).max()}
    d.update({f"hidden_states[{i}]": fr.rel_dist(x[i], o["hidden_states"][i]).max() for i in x})
    return d


def test_conversion_round_trip(dino):
    """weights_in and weights_out land as fc1 [2 F][D] and fc2 [D][F] unchanged, in HF's x1 | x2 order; the file says "swiglu"."""
    geo, classifier, m, _, path, vf, _, _ = dino
    R, L = do.GEOMETRIES[geo][5], 2
    assert m.config.use_swiglu_ffn
    assert (vf.layer_scale, vf.reg_tokens, vf.pool, vf.activation) == (1, R, "cls_patch_mean" if classifier else "token", "swiglu")
    assert b"swiglu" in open(path, "rb").read()
    assert len(vf.tensors) == 4 + 12 * L + 4 + 2 * L + (R > 0)
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    pre = {"micro": "dinov2.", "micro_reg": "dinov2_with_registers."}[geo] if classifier else ""
    for i in range(L):
        h = f"{pre}encoder.layer.{i}.mlp."
        assert vf.tensors[f"blocks.{i}.mlp.fc1.weight"].shape == (2 * F, D) and vf.tensors[f"blocks.{i}.mlp.fc2.weight"].shape == (D, F)
        assert np.array_equal(np.asarray(vf.tensors[f"blocks.{i}.mlp.fc1.weight"], np.float32), sd[h + "weights_in.weight"])
        assert np.array_equal(vf.tensors[f"blocks.{i}.mlp.fc1.bias"], sd[h + "weights_in.bias"])
        assert np.array_equal(np.asarray(vf.tensors[f"blocks.{i}.mlp.fc2.weight"], np.float32), sd[h + "weights_out.weight"])
        assert np.array_equal(vf.tensors[f"blocks.{i}.mlp.fc2.bias"], sd[h + "weights_out.bias"])
    assert not any("weights_in" in k or "weights_out" in k for k in vf.tensors)


def test_emulation_matches_the_hf_oracle(dino):
    geo, classifier, _, _, _, vf, imgs, o = dino
    d = _distances(vf, imgs, o)
    print(geo, classifier, {k: f"{v:.2e}" for k, v in d.items()})
    assert max(d.values()) <= EMU_BOUND, d


def test_swapped_halves_fail_the_oracle_check(dino):
    """silu on x2 instead of x1 (fc1's halves swapped) lands far outside the bound the right order meets."""
    _, _, _, _, _, vf, imgs, o = dino
    bad = copy.deepcopy(vf)
    for i in range(vf.num_hidden_layers):
        for k in ("weight", "bias"):
            n = f"blocks.{i}.mlp.fc1.{k}"
            bad.tensors[n] = np.concatenate(np.split(np.asarray(vf.tensors[n]), 2, axis=0)[::-1], axis=0)
    worst = max(_distances(bad, imgs, o).values())
    print(f"halves swapped: {worst:.2e}")
    assert worst > 10 * EMU_BOUND


def test_converter_refuses_a_swiglu_config_without_swiglu_weights(tmp_path):
    m = do.build_hf("micro", True)
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    with pytest.raises(ValueError, match="use_swiglu_ffn"):
        cv.dinov2_to_model_file(sd, {"num_attention_heads": 2, "use_swiglu_ffn": True}, str(tmp_path / "x.gguf"))


def test_swiglu_config_ignores_hidden_act_and_mlp_ratio(dino, tmp_path):
    """HF's SwiGLU FFN reads neither hidden_act nor mlp_ratio; F comes from the tensors."""
    geo, classifier, m, _, path, vf, _, _ = dino
    if not (geo == "micro" and classifier):
        pytest.skip("one class is enough")
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    out = str(tmp_path / "x.gguf")
    cv.dinov2_to_model_file(sd, {"num_attention_heads": 2, "use_swiglu_ffn": True, "hidden_act": "relu", "mlp_ratio": 3}, out,
                            img_size=do.image_size(geo))
    back = gf.read_gguf(out)
    assert back.activation == "swiglu"
    for k, a in vf.tensors.items():
        assert np.array_equal(np.asarray(back.tensors[k]), np.asarray(a)), k


def _create(vf, arch, edit=None):
    """vitb200_create_arch on no GPU: every refusal below comes before the device check."""
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
    eng._check(eng.lib().vitb200_create_arch(C.byref(hp), C.byref(arch), ts, len(entries), 0, 2, 1, 0, C.byref(h)), "vitb200_create_arch")


def _resize(name, rows, cols):
    """An edit that replaces tensor `name` by a [rows][cols] one of its type."""
    def edit(es):
        return [(n, np.zeros((rows, cols), a.dtype), ft) if n == name else (n, a, ft) for n, a, ft in es]
    return edit


def test_engine_refusals_need_no_gpu(dino):
    geo, classifier, _, _, _, vf, _, _ = dino
    R, pool = vf.reg_tokens, int(classifier)
    ok = lambda **kw: eng.Arch(**dict(dict(pre_norm=0, activation=4, layer_scale=1, reg_tokens=R, pool=pool), **kw))
    cases = [(ok(activation=5), "vitb200_arch.activation = 5 out of range"),
             (ok(pool=2, reg_tokens=0), "vitb200_arch.activation = 4 out of range for pool 2"),
             (ok(pool=3, reg_tokens=0), "vitb200_arch.activation = 4 out of range for pool 3")]
    for arch, msg in cases:
        with pytest.raises(eng.VitB200Error, match=msg):
            _create(vf, arch)
    edits = [(_resize("blocks.0.mlp.fc1.weight", 2 * F + 1, D), "even row count 2 F in 'blocks.0.mlp.fc1.weight', got 689"),
             (_resize("blocks.0.mlp.fc1.weight", 2 * 340, D), "F = 340 is not a multiple of 8"),
             (_resize("blocks.0.mlp.fc1.weight", 2 * (8 * D + 8), D), r"F = 1032 out of range \(8..1024 = 8 D\)"),
             (_resize("blocks.1.mlp.fc1.weight", 2 * (F + 8), D), "block 1's mlp.fc1 .* disagrees with F = 344"),
             (_resize("blocks.1.mlp.fc2.weight", D, F - 8), "block 1's mlp.fc1 .* disagrees with F = 344"),
             (_resize("blocks.0.mlp.fc2.weight", D, F + 8), "block 0's mlp.fc1 .* disagrees with F = 344")]
    for edit, msg in edits:
        with pytest.raises(eng.VitB200Error, match=msg):
            _create(vf, ok(), edit=edit)
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(eng.VitB200Error, match="no CPU fallback"):
            _create(vf, ok())                               # everything else is in order: the device check is next


def test_gguf_activation_key(tmp_path):
    """"swiglu" round-trips through write_gguf / read_gguf; a reference file carries no vit.activation."""
    vf = gf.read(model_path("micro", "f16"))
    vf.activation = "swiglu"
    p = str(tmp_path / "s.gguf")
    gf.write_gguf(p, vf)
    assert gf.read_gguf(p).activation == "swiglu"
    assert gf.ARCH_ACTIVATIONS.index("swiglu") == 4
    vf.activation = "swish"
    with pytest.raises(ValueError, match="unknown activation 'swish'"):
        gf.write_gguf(str(tmp_path / "t.gguf"), vf)


def test_gguf_parser_fuzzed_with_a_swiglu_file(dino, tmp_path):
    """tests/cpp/gguf_fuzz.cpp under ASan / UBSan with a SwiGLU DINOv2 file (vit.activation "swiglu") as its GGUF seed."""
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
    assert b"swiglu" in open(path, "rb").read()
    r = subprocess.run([exe, path, model_path("micro", "f16")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert r.stdout.count("rejected") == 2
