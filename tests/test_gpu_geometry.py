"""The forward pass at every geometry the engine selects a kernel or a launch path by (gf.CONFIGS, 2-layer models):

    p8        P 8, 785 tokens      patchify<8,3>; MMA8 attention (641 <= N <= 896); bulk LayerNorm NV 3; patch rows alias the MLP buffer
    p32       P 32, 145 tokens     patchify<32,3>; patch GEMM K = 3072 on the 6-stage ring; own patch buffer; NV 4; wgmma attention
    d640      D 640, 257 tokens    bulk LayerNorm NV 5; MMA16 attention; proj with 5 column tiles
    d896p14   D 896, P 14          bulk LayerNorm NV 7; patchify<14,3> with K padded 588 -> 640
    d320      D 320                D % 128 = 64: block LayerNorms on the row-per-warp kernel; odd tile counts in qkv and proj
    d1536     D 1536               row-per-warp LayerNorm MAXV 16 everywhere; fc2 K = 6144
    d2048     D 2048, 1 layer      the largest accepted hidden size: 16 float4 per lane
    d64       D 64, 1 head         half a 128-column tile in proj and head; 16 of 32 lanes live in the LayerNorm
    vitstr_p8 1 channel, P 8       patchify<8,1>; grayscale preprocess and recognition at P 8

Each is checked against the C restatement (bit-exact against the compiled reference at these geometries: tests/test_oracle.py), per
layer through the debug taps and end to end, for batch invariance across the CUDA-graph path, for the u8 entry point and on the FP8
engine."""
import numpy as np
import pytest

from tests.util import pkg, gf, model_path
from tests.test_gpu_forward import check_parity, rel_err
from tests.test_gpu_fp8 import E2E_TOL
from tests import fp8_reference as fr
from tests.emulation import Emulation
from oracle import restatement as rs

eng = pkg.engine
pytestmark = pytest.mark.gpu

RGB = ["p8", "p32", "d640", "d896p14", "d320", "d1536", "d2048", "d64"]
GEOMETRIES = RGB + ["vitstr_p8"]
# per-tap tolerances of test_gpu_forward.py::test_taps_match_restatement, relative to the tap's largest magnitude
TAP_TOL = [("embed", 1e-5), ("ln1", 2e-3), ("qkv", 2e-3), ("attn", 2e-3), ("x1", 2e-3), ("ln2", 2e-3), ("h", 3e-3), ("x2", 2e-3),
           ("final_ln", 3e-3), ("x_final", 2e-3)]


def _setup(cfg, n=3, seed=5):
    path = model_path(cfg, "f16")
    vf = gf.read(path)
    ht = 25 if cfg.startswith("vitstr") else 1
    imgs = (gf.synthetic_gray_images if ht > 1 else gf.synthetic_images)(n, vf.img_size, seed=seed)
    return path, vf, ht, imgs


def _launches(cfg):
    return 3 + 7 * gf.CONFIGS[cfg][1] + 3


@pytest.mark.parametrize("cfg", GEOMETRIES)
def test_taps_match_restatement(cfg):
    """Every intermediate of the first and the last block.  The embed tap at 1e-5 is the sharp check of patchify, the patch GEMM, its
    epilogue (bias + position embedding) and the zeroed K padding."""
    path, vf, ht, imgs = _setup(cfg, 2, seed=7)
    om = rs.OracleModel(vf, gf.tensor_specs, head_tokens=ht)
    rs.set_threads(8)
    m = eng.vit_model_load(path, 0, 2, head_tokens=ht)
    names = [n for n, _ in TAP_TOL if ht == 1 or n != "final_ln"]   # the oracle's final_ln tap is one pooled row
    worst = {}
    for layer in sorted({0, vf.num_hidden_layers - 1}):
        _, _, taps = eng.vit_predict_debug(m, imgs, layer, taps=tuple(names))
        for b in range(2):
            _, _, t_o = om.forward(imgs[b], layer, tuple(names))
            for name, tol in TAP_TOL:
                if name in names:
                    r = t_o[name]
                    d = float(np.abs(taps[name][b] - r).max() / np.abs(r).max())
                    worst[(layer, name)] = max(worst.get((layer, name), 0.0), d)
    m.close()
    om.close()
    print(cfg, {f"{k[0]}:{k[1]}": f"{v:.2e}" for k, v in worst.items()})
    tol = dict(TAP_TOL)
    bad = {k: v for k, v in worst.items() if v > tol[k[1]]}
    assert not bad, bad


@pytest.mark.parametrize("cfg", RGB)
def test_logits_match_restatement(cfg):
    """Up to 224 tokens q, k and v are split-precision (hi + lo f16) and the 2-layer micro models' bounds apply; beyond, q, k and v are
    f16 and the bounds of test_long_sequence_geometry_vit_large_384 apply.  Top-1 must match wherever the reference's top-2 gap is clear."""
    path, vf, ht, imgs = _setup(cfg)
    om = rs.OracleModel(vf, gf.tensor_specs)
    rs.set_threads(8)
    p_ref, l_ref = om.forward_batch(imgs)
    om.close()
    m = eng.vit_model_load(path, 0, 3)
    probs, idx, val, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    m.close()
    re = rel_err(logits, l_ref)
    l2 = np.linalg.norm(logits - l_ref, axis=1) / np.linalg.norm(l_ref, axis=1)
    print(f"{cfg} (N = {vf.n_tokens}): max-norm {np.array2string(re, precision=6)}, L2 {np.array2string(l2, precision=6)}")
    if vf.n_tokens <= 224:
        check_parity(logits, probs, idx, l_ref, p_ref, max_tol=1.5e-3)
    else:
        assert re.max() <= 2e-3, re
        assert l2.max() <= 1e-3, l2
    top2 = np.sort(l_ref, axis=1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 2.5 * np.abs(logits - l_ref).max(axis=1)
    assert (logits.argmax(1) == l_ref.argmax(1))[clear].all()
    assert np.array_equal(val, np.take_along_axis(probs, idx.astype(np.int64), 1))


@pytest.mark.parametrize("cfg", GEOMETRIES)
def test_batch_invariance_and_graph_path(cfg):
    """Each image alone -- eager, graph capture, graph replay -- gives the logits it gets in the 3-image batch, bit for bit, with the fixed
    launch count 3 + 7 L + 3."""
    path, vf, ht, imgs = _setup(cfg, seed=11)
    m = eng.vit_model_load(path, 0, 3, head_tokens=ht)
    l_all = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    assert m.last_launch_count() == _launches(cfg)
    assert np.isfinite(l_all).all()
    for b in range(3):
        for rep in range(3):
            l = eng.vit_predict(m, imgs[b:b + 1], 5, want_logits=True)[3]
            assert np.array_equal(l[0], l_all[b]), (b, rep)
            assert m.last_launch_count() == _launches(cfg)
    m.close()


@pytest.mark.parametrize("cfg", RGB)
def test_u8_path_writes_the_patch_rows_patchify_writes(cfg):
    """The u8 preprocess writes the f16 patch matrix itself (no patchify): its logits equal those of the f32 images it returns, through
    patchify, bit for bit."""
    path, vf, ht, _ = _setup(cfg)
    rng = np.random.default_rng(3)
    u8 = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((97, 131), (300, 277), (vf.img_size + 1, vf.img_size - 3))]
    m = eng.vit_model_load(path, 0, 3)
    for bilinear in (False, True):
        f32, probs, idx, val, logits = eng.vit_image_preprocess_predict(m, u8, bilinear=bilinear)
        l32 = eng.vit_predict(m, f32, 5, want_logits=True)[3]
        assert np.array_equal(logits, l32), bilinear
    m.close()


@pytest.mark.parametrize("cfg", GEOMETRIES)
def test_fp8_engine(cfg):
    """The e4m3 LayerNorms (bulk-copy NV 2-7, row-per-warp up to MAXV 16) through the ln1 / ln2 taps of the first and last block, as in
    test_gpu_fp8.py::test_taps_are_the_dequantised_layernorm_rows, and the logits against the emulation of the recipe."""
    path, vf, ht, imgs = _setup(cfg)
    m = eng.vit_model_load(path, 0, 3, head_tokens=ht, fp8=True)
    assert m.fp8
    D, t = vf.hidden_size, vf.tensors
    for layer in sorted({0, vf.num_hidden_layers - 1}):
        _, _, taps = eng.vit_predict_debug(m, imgs, layer, taps=("ln1", "x1", "ln2") + (("embed",) if layer == 0 else ("x2",)))
        if layer == 0:
            x_in = taps["embed"]
        else:
            x_in = eng.vit_predict_debug(m, imgs, layer - 1, taps=("x2",))[2]["x2"]
        for name, x, wn in (("ln1", x_in, "norm1"), ("ln2", taps["x1"], "norm2")):
            y = rs.layernorm(x.reshape(-1, D), np.asarray(t[f"blocks.{layer}.{wn}.weight"], np.float32),
                             np.asarray(t[f"blocks.{layer}.{wn}.bias"], np.float32))
            q, sa = fr.quantize_rows(y)
            want = fr.e4m3_value(q) * sa[:, None]
            got = taps[name].reshape(-1, D)
            assert (np.abs(got - want) <= 5e-7 * np.abs(want)).mean() > 0.99, (layer, name)
            assert np.abs(got - want).max() <= np.abs(want).max() / 8, (layer, name)
    logits = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    m.close()
    emu = Emulation(vf, head_tokens=ht).forward(imgs)
    d = fr.rel_dist(logits, emu)
    print(f"{cfg} FP8: GPU vs emulation {np.array2string(d, precision=4)} (bound {E2E_TOL:.4f})")
    assert d.max() <= E2E_TOL, d


def test_vitstr_p8_logits_and_recognition():
    """The grayscale model at P 8 against the restatement (head_tokens 25, the bounds of
    test_gpu_forward.py::test_vitstr_extension_matches_the_reference), and recognition from u8 -- the grayscale preprocess writing P 8
    patch rows -- equal to the preprocess followed by the f32 forward, on both engines."""
    path, vf, ht, imgs = _setup("vitstr_p8")
    om = rs.OracleModel(vf, gf.tensor_specs, head_tokens=25)
    rs.set_threads(8)
    p_ref, l_ref = om.forward_batch(imgs)
    om.close()
    m = eng.vit_model_load(path, 0, 4, head_tokens=25)
    probs, idx, val, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    n = imgs.shape[0]
    lf, rf = logits.reshape(n, -1), l_ref.reshape(n, -1)
    re = np.abs(lf - rf).max(1) / np.abs(rf).max(1)
    l2 = np.linalg.norm(lf - rf, axis=1) / np.linalg.norm(rf, axis=1)
    print(f"vitstr_p8: max-norm {np.array2string(re, precision=6)}, L2 {np.array2string(l2, precision=6)}")
    assert np.median(re) <= 1e-3 and re.max() <= 1.5e-3, re
    assert (l2 <= 1.25e-3).all(), l2
    top2 = np.sort(l_ref, -1)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 2.5 * np.abs(logits - l_ref).max(-1)
    assert clear.mean() > 0.9 and (idx[..., 0] == l_ref.argmax(-1))[clear].all()
    m.close()
    rng = np.random.default_rng(2)
    u8 = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((32, 100), (65, 63), (7, 300), (64, 64))]
    for fp8 in (False, True):
        m = eng.vit_model_load(path, 0, 4, head_tokens=25, fp8=fp8)
        texts, scores, chars, lengths, pr = eng.vitstr_recognize_u8(m, u8, probs=True)
        gray = eng.vitstr_preprocess_u8(m, u8)
        p2 = eng.vit_predict(m, gray, 1)[0]
        assert np.array_equal(pr, p2), fp8
        am = p2[:, 1:].argmax(axis=2)
        for b in range(len(u8)):
            k = int(lengths[b])
            assert np.array_equal(chars[b, :k], am[b, :k]), (fp8, b)
            assert k == 24 or am[b, k] == 1, (fp8, b)
            assert (chars[b, k:] == -1).all()
            assert np.isclose(scores[b], np.prod(p2[b, 1:k + 1].max(axis=1).astype(np.float64)), rtol=1e-12, atol=0)
        m.close()
