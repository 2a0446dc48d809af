"""The FP8 engine's host side, without a GPU: argument checks of the new entry points, the upload-time weight quantisation against
torch's e4m3, and the accuracy cost of the FP8 recipe measured on its numpy emulation (tests/emulation.py) against the
reference's golden logits."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from tests.util import pkg, gf, model_path
from tests import fp8_reference as fr
from tests.emulation import Emulation

eng = pkg.engine
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# Max-norm logit distance per image, max |FP8 emulation - golden| / max |golden|, over the fixtures below: the accuracy cost of
# the recipe (README.md).  Measured 0.050-0.115; the f16 engine's own emulation sits at <= 1.2e-3 from the same golden logits.
FP8_COST_MAX = 0.13
# The emulation against itself with f64 instead of f32 accumulation: a last-bit change of a LayerNorm output moves some values
# across an e4m3 rounding boundary (one e4m3 step is 6-12 % of the value), and the flips compound over the blocks.  Measured
# 1.1e-4 (micro, 2 blocks), 0.024 (tiny), 0.027 (tiny q8_0), 0.037 (base).  tests/test_gpu_fp8.py sets its end-to-end tolerance
# from this floor: the GPU accumulates in yet another order, so it differs from the emulation by about the same amount.
FP8_FLOOR_MAX = 0.045


def _last_error():
    return eng.lib().vitb200_last_error().decode()


def test_null_and_bad_arguments_are_rejected():
    L = eng.lib()
    h = C.c_void_p()
    hp = eng.Hparams(768, 12, 12, 1000, 16, 224, 1, 1e-6)
    assert L.vitb200_create_fp8(None, None, 0, 0, 1, 1, C.byref(h)) != 0 and "null" in _last_error()
    assert L.vitb200_create_fp8(C.byref(hp), None, 0, 0, 1, 1, C.byref(h)) != 0
    assert L.vitb200_create_fp8(C.byref(hp), None, 0, 0, 1, 1, None) != 0
    assert L.vitb200_create_from_file_fp8(None, 0, 1, 1, C.byref(h)) != 0
    assert L.vitb200_create_from_file_fp8(b"/nonexistent/model.bin", 0, 1, 1, C.byref(h)) != 0
    assert not h.value
    assert L.vitb200_fp8(None) == 0
    w = np.zeros(8, np.float16)
    q = np.zeros(8, np.uint8)
    s = C.c_float()
    assert L.vitb200_test_quantize_fp8(None, 8, q.ctypes.data, C.byref(s)) != 0
    assert L.vitb200_test_quantize_fp8(w.ctypes.data, 8, None, C.byref(s)) != 0
    assert L.vitb200_test_quantize_fp8(w.ctypes.data, 8, q.ctypes.data, None) != 0
    assert L.vitb200_test_quantize_fp8(w.ctypes.data, 0, q.ctypes.data, C.byref(s)) != 0
    a = np.zeros(64 * 64, np.uint8)
    f = np.zeros(64 * 64, np.float32)
    assert L.vitb200_test_gemm_fp8(0, 64, 64, 64, 0, None, f.ctypes.data, a.ctypes.data, 1.0, f.ctypes.data, f.ctypes.data) != 0
    assert L.vitb200_test_gemm_fp8(0, 64, 64, 64, 0, a.ctypes.data, None, a.ctypes.data, 1.0, f.ctypes.data, f.ctypes.data) != 0
    for epi in (eng.EPI_BIAS_RESID_F32, eng.EPI_PATCH_F32, eng.EPI_BIAS_F32, 5):  # f32-output epilogues have no e4m3 form; 5 is none
        assert L.vitb200_test_gemm_fp8(0, 64, 64, 64, epi, a.ctypes.data, f.ctypes.data, a.ctypes.data, 1.0, f.ctypes.data,
                                       f.ctypes.data) != 0 and "epilogue" in _last_error()
    assert L.vitb200_test_gemm_fp8(0, 64, 64, 40, 0, a.ctypes.data, f.ctypes.data, a.ctypes.data, 1.0, f.ctypes.data, f.ctypes.data) != 0
    assert L.vitb200_test_layernorm_fp8(0, 4, 64, None, f.ctypes.data, f.ctypes.data, 1e-6, a.ctypes.data, f.ctypes.data) != 0
    assert L.vitb200_test_layernorm_fp8(0, 4, 64, f.ctypes.data, f.ctypes.data, f.ctypes.data, 1e-6, None, f.ctypes.data) != 0
    assert L.vitb200_test_layernorm_fp8(0, 4, 60, f.ctypes.data, f.ctypes.data, f.ctypes.data, 1e-6, a.ctypes.data, f.ctypes.data) != 0


FP8_WIDTH = "FP8 engine: hidden size 72 not supported \\(a multiple of 16: the e4m3 activation rows of D bytes are read in 16-byte strides"


def test_fp8_image_towers_need_hidden_sizes_of_16_byte_rows(tmp_path):
    """A SigLIP-pooled image tower with one 72-column head (D = 72): the f16 engine takes it; the FP8 engine's e4m3 rows would be 72 bytes,
    which its TMA maps cannot stride, so it is refused before the device is touched, naming the limit."""
    path = str(tmp_path / "m.bin")
    gf.write_synthetic(path, (72, 1, 1, 16, 64), 1)
    vf = gf.read(path)
    vf.pool = "mean"  # head dim 72 runs with the SigLIP pools only: patch rows, no class token
    del vf.tensors["cls_token"]
    vf.tensors["pos_embed"] = np.ascontiguousarray(np.asarray(vf.tensors["pos_embed"]).reshape(-1, 72)[1:][None])
    with pytest.raises(eng.VitB200Error, match=FP8_WIDTH):
        eng.vit_model_from_tensors(vf, 0, 2, fp8=True)
    if torch.cuda.is_available():
        eng.vit_model_from_tensors(vf, 0, 2).close()
    else:
        with pytest.raises(eng.VitB200Error, match="no CUDA device"):
            eng.vit_model_from_tensors(vf, 0, 2)


def test_fp8_text_towers_need_hidden_sizes_of_16_byte_rows():
    """A SigLIP text tower with one 72-column head is refused in its FP8 form before the device is touched; with two heads (D = 144) the
    width passes and the load goes on to the next check (here: the blocks this stub lacks)."""
    L = eng.lib()
    for D, heads in ((72, 1), (144, 2)):
        tok = np.zeros((8, D), np.float16)
        ts = (eng.Tensor * 1)()
        ts[0].name, ts[0].data, ts[0].type, ts[0].n_dims = b"token_embd.weight", tok.ctypes.data, 1, 2
        ts[0].ne[0], ts[0].ne[1], ts[0].ne[2], ts[0].ne[3] = D, 8, 1, 1
        hp = eng.Hparams(D, 1, heads, 96, 0, 0, 1, 1e-6)
        ta = eng.TextArch(16, 0, 2, 2, gf.ARCH_ACTIVATIONS.index("gelu_pytorch_tanh"), float("nan"), float("nan"))
        h = C.c_void_p()
        assert L.vitb200_create_text(C.byref(hp), C.byref(ta), ts, 1, 0, 2, 1, C.byref(h)) != 0 and not h.value
        if D == 72:
            assert re.search(FP8_WIDTH, _last_error()), _last_error()
        else:
            assert "FP8 engine" not in _last_error() and "hidden size" not in _last_error(), _last_error()


def _torch_e4m3(w16, scale_inv):
    t = torch.from_numpy(np.asarray(w16, np.float16).astype(np.float32)) * torch.tensor(np.float32(scale_inv))
    # torch turns values above 464 into NaN instead of saturating: the scaling keeps every value at 448 to within the f32 rounding of
    # amax * (448 / amax), which e4m3 rounds back to 448
    assert float(t.abs().max()) <= 448.0 * (1 + 2.0 ** -22)
    return t.to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def _check_quantize(w16):
    q, s = eng.test_quantize_fp8(w16)
    amax = np.float32(np.abs(np.asarray(w16, np.float16).astype(np.float32)).max())
    if amax == 0:
        assert s == 1.0 and not q.any()
        return
    assert np.float32(s) == amax / np.float32(448)
    assert np.array_equal(q, _torch_e4m3(w16, np.float32(448) / amax))


@pytest.mark.parametrize("seed,scale", [(0, 0.02), (1, 1.0), (2, 300.0), (3, 1e-3)])
def test_quantize_matches_torch_on_random_tensors(seed, scale):
    rng = np.random.default_rng(seed)
    _check_quantize((rng.standard_normal(50_000) * scale).astype(np.float16))


def test_quantize_matches_torch_on_fixture_weights():
    vf = gf.read(model_path("tiny", "f16"))
    for i in (0, 11):
        for name in ("attn.qkv.weight", "mlp.fc1.weight"):
            _check_quantize(np.asarray(vf.tensors[f"blocks.{i}.{name}"], np.float16))


def test_quantize_edge_cases():
    _check_quantize(np.zeros(1000, np.float16))  # all zero: scale 1, all codes zero
    sub = np.array([0, 2.0 ** -24, -3 * 2.0 ** -24, 2.0 ** -20, -(2.0 ** -15)], np.float32).astype(np.float16)  # amax an f16 subnormal
    assert np.abs(sub.astype(np.float32)).max() < 2.0 ** -14
    _check_quantize(sub)
    _check_quantize(np.array([65504, -65504, 1, -1e-3], np.float16))


def test_emulation_rows_match_the_tensor_rule():
    """quantize_rows (the LayerNorm's per-row rule) and quantize_tensor (the weights' rule) agree on a single row."""
    rng = np.random.default_rng(5)
    y = rng.standard_normal((1, 300)).astype(np.float32).astype(np.float16)
    q1, s1 = fr.quantize_rows(y.astype(np.float32))
    q2, s2 = fr.quantize_tensor(y)
    assert np.array_equal(q1, q2) and s1[0] == s2
    assert np.array_equal(q2, eng.test_quantize_fp8(y)[0])


@pytest.mark.parametrize("cfg,ftype", [("micro", "f16"), ("tiny", "f16"), ("tiny", "q8_0"), ("base", "f16")])
def test_emulated_accuracy_cost_and_floor(cfg, ftype):
    g = np.load(os.path.join(GOLD, f"{cfg}_{ftype}.npz"))
    vf = gf.read(model_path(cfg, ftype))
    imgs = gf.synthetic_images(int(g["n_images"]), vf.img_size, seed=int(g["image_seed"]))
    f16 = Emulation(vf, fp8=False).forward(imgs)
    e32 = Emulation(vf).forward(imgs)
    e64 = Emulation(vf, acc=np.float64).forward(imgs)
    # the emulation's f16 form reproduces the golden logits as closely as the f16 engine does: the shared pieces are right
    assert fr.rel_dist(f16, g["logits"]).max() <= (2e-2 if ftype == "q8_0" else 1.5e-3)
    cost = fr.rel_dist(e32, g["logits"])
    floor = fr.rel_dist(e32, e64)
    print(f"{cfg} {ftype}: FP8 cost {np.round(cost, 4)}, f32-vs-f64 floor {floor.max():.2e}")
    assert cost.max() <= FP8_COST_MAX
    assert floor.max() <= FP8_FLOOR_MAX
