"""The FP8 engine on the GPU: the e4m3 GEMM element by element, the e4m3 LayerNorm against the emulation, end-to-end logits against
the emulation of the recipe (tests/emulation.py), and every entry point on an FP8 engine."""
import math
import os

import numpy as np
import pytest

from tests.util import pkg, gf, model_path
from tests import fp8_reference as fr
from tests.emulation import Emulation
from tests.test_fp8_abi import FP8_FLOOR_MAX
from tests import test_gpu_gemm_schedule as gs
from oracle import restatement as rs

eng = pkg.engine
pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BM = BN = 128

# End-to-end tolerance, max |GPU - emulation| / max |emulation| per image: twice the emulation's own f32-vs-f64 accumulation floor
# (FP8_FLOOR_MAX, tests/test_fp8_abi.py).  The GPU sums in a third order and its LayerNorm in f32 rather than double, so its e4m3
# rounding flips are of the same kind and size as the floor's.
E2E_TOL = 2 * FP8_FLOOR_MAX


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- GEMM, exact ---------------------------------------------------------------------------------------------------------------
def _check_exact(M, N, K, epi, seed):
    """Small-integer e4m3 operands (|v| <= 4, exact in e4m3) with power-of-two scales: A is sparse enough that sum_k |a| |w| < 2^11 on
    every row, so every partial sum is an integer below 2^11 and the result does not depend on the accumulator's width or order.
    Epilogues 7, 8, 10 and 11 also get -1e4 in every TAIL_EVERY-th bias column (of x1 for SwiGLU), and are checked as functions of x
    (of the pair x1, x2), as in test_gpu_gemm_schedule.py: x is a multiple of 1/8 (scales 1/8 .. 1/2)."""
    rng = np.random.default_rng(seed)
    keep = min(1.0, 96.0 / K)
    A = rng.integers(-2, 3, size=(M, K)) * (rng.random((M, K)) < keep)
    W = rng.integers(-4, 5, size=(N, K))
    assert (np.abs(A).sum(axis=1) * 4 < 2 ** 11).all()
    sa = (2.0 ** rng.integers(-1, 2, size=M)).astype(np.float32)
    sw = np.float32(0.25)
    bias = rng.integers(-8, 9, size=N).astype(np.float32)
    if epi in gs.NEW:
        bias[:N // 2 if epi == eng.EPI_SWIGLU else N:gs.TAIL_EVERY] = -1e4
    out = eng.test_gemm_fp8(M, N, K, epi, fr.e4m3_bits(A), sa, fr.e4m3_bits(W), sw, bias)
    acc = A.astype(np.float64) @ W.astype(np.float64).T  # BLAS in f64 on integers below 2^11: exact
    x = (acc * (sa[:, None].astype(np.float64) * sw) + bias).astype(np.float32)  # exact: at most 11 + 4 significant bits (17 with -1e4)
    if epi in gs.NEW:
        q = (x.astype(np.float64) * 8).astype(np.int64)
        assert np.array_equal(q / 8, x)
        if epi == eng.EPI_SWIGLU:
            assert out.shape == (M, N // 2)
            want = gs.check_swiglu(out, q[:, :N // 2], q[:, N // 2:], 0.125)
        else:
            want = gs.check_activation(out, q, 0.125, epi)
        return gs.assert_same_bits(out, want)
    if epi == eng.EPI_BIAS_F16_HILO:
        want = x  # hi + lo carries 22 bits
    elif epi == eng.EPI_BIAS_F16:
        want = x.astype(np.float16).astype(np.float32)
    elif epi == eng.EPI_BIAS_GELU_F16:
        # as in test_gpu_gemm_schedule.py: each output a function of its f16 pre-activation, within one f16 ulp of the table
        x16 = x.astype(np.float16).astype(np.float32)
        q = (x16 * 8).astype(np.int64)  # f16 rounds a multiple of 1/8 below 2^11 to another one
        assert np.array_equal(q / 8, x16)
        want, seen, per_value = gs.function_of(out, q - q.min())
        table = rs.gelu_table(((seen + q.min()) / 8).astype(np.float32))
        ulp = np.maximum(np.abs(table), 2.0 ** -14) * 2.0 ** -10
        assert (np.abs(per_value - table) <= ulp).all()
    else:
        raise ValueError(epi)
    bad = out != want
    if bad.any():
        r, c = np.argwhere(bad)[0]
        tiles = sorted({(int(i) // BM, int(j) // BN) for i, j in np.argwhere(bad)[:100000]})
        raise AssertionError(f"{int(bad.sum())} of {bad.size} elements differ; first at row {r} col {c}: {out[r, c]} != {want[r, c]}; "
                             f"tiles (m, n) {tiles[:8]}")


@pytest.mark.parametrize("epi", [eng.EPI_BIAS_F16, eng.EPI_BIAS_GELU_F16, eng.EPI_BIAS_F16_HILO, eng.EPI_BIAS_GELU_ERF_F16,
                                 eng.EPI_BIAS_QUICK_GELU_F16, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16, eng.EPI_SWIGLU])
@pytest.mark.parametrize("K", [64, 192, 768, 1024, 3072, 144, 160, 208, 240, 400, 1040])
def test_gemm_exact_ragged_m(epi, K):
    """M ends inside a tile's second 64-row half; K = 64 is a partial k-block (zero-filled), 3072 runs the 6-slot ring.  K = 144, 160,
    208, 240, 400 and 1040 end in a k-block of 128 that holds 16, 32, 80, 112, 16 and 16 columns of K (the rest zero-filled): D = 80 H
    with H = 2, 3, 5, 13, and the So400m micro towers' 144.  SwiGLU: F = 192, 3 column tiles, the last pair's second tile past N."""
    _check_exact(197 * 7, 384, K, epi, seed=K + epi)


@pytest.mark.parametrize("per_cluster,extra", [(3, 0), (3, 1), (4, -1)])
@pytest.mark.parametrize("K,epi", [(192, eng.EPI_BIAS_F16), (768, eng.EPI_BIAS_F16_HILO), (3072, eng.EPI_BIAS_GELU_F16),
                                   (192, eng.EPI_BIAS_GELU_ERF_F16), (3072, eng.EPI_BIAS_GELU_ERF_F16), (320, eng.EPI_BIAS_QUICK_GELU_F16),
                                   (2048, eng.EPI_BIAS_QUICK_GELU_F16), (192, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16),
                                   (3072, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16), (192, eng.EPI_SWIGLU), (3072, eng.EPI_SWIGLU),
                                   (400, eng.EPI_BIAS_F16_HILO), (208, eng.EPI_BIAS_F16), (240, eng.EPI_BIAS_GELU_F16)])
def test_gemm_exact_tile_counts_around_the_grid(per_cluster, extra, K, epi):
    """As in test_gpu_gemm_schedule.py; SwiGLU with F = 128, one pair per row band.  K = 400, 208 and 240: 4, 2 and 2 k-blocks, the last
    one partly zero-filled."""
    pairs = per_cluster * (_sms() // 2) + extra
    _check_exact(pairs * BM, 2 * BN, K, epi, seed=pairs + K)


@pytest.mark.parametrize("epi", [eng.EPI_BIAS_GELU_ERF_F16, eng.EPI_BIAS_QUICK_GELU_F16, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16, eng.EPI_SWIGLU])
def test_gemm_exact_warpgroups_take_different_column_tiles(epi):
    """As test_gpu_gemm_schedule.py::test_warpgroups_take_different_column_tiles: a pair count coprime to the cluster count, so the two
    warpgroups of a CTA run different column tiles (and read their own bias and row scales)."""
    n_pairs = next(n for n in (5, 7, 11, 13) if math.gcd(n, _sms() // 2) == 1)
    _check_exact(197 * 63, 2 * BN * n_pairs, 3072, epi, seed=n_pairs + epi)


@pytest.mark.parametrize("N,K,epi", [(2304, 768, eng.EPI_BIAS_F16_HILO), (3072, 768, eng.EPI_BIAS_GELU_F16),
                                     (3072, 768, eng.EPI_BIAS_GELU_ERF_F16), (3072, 768, eng.EPI_BIAS_QUICK_GELU_F16),
                                     (3072, 768, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16), (2 * 4096, 1536, eng.EPI_SWIGLU)])
def test_gemm_exact_vit_b_shapes(N, K, epi):
    """qkv and fc1 of ViT-B/16 at batch 256 (tanh GELU with the f16 table, erf, QuickGELU, PyTorch's tanh GELU); ViT-g's SwiGLU fc1
    (F = 4096) at batch 64 with 4 registers (261 tokens)."""
    _check_exact(64 * 261 if epi == eng.EPI_SWIGLU else 256 * 197, N, K, epi, seed=N + K)


@pytest.mark.parametrize("M,N,K,epi", [(M, N, K, epi) for M, N, K, epi in gs.TOWER_LAYERS if epi != eng.EPI_BIAS_RESID_F32])
def test_gemm_exact_tower_layer_shapes(M, N, K, epi):
    """The FP8 engine's qkv and fc1 of SigLIP So400m (3 x 729 tokens; fc1's last column tile 80 columns wide) and ViT-H/14 (3 x 257)."""
    _check_exact(M, N, K, epi, seed=M + N + K + epi)


# ---- GEMM, random operands -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [768, 3072])
def test_gemm_random_against_f64(K):
    """Random e4m3 operands against an f64 sum.  The error is reported relative to sum_k |a w| of the element (the condition-free
    scale of the sum).  f32 accumulation would stay near K 2^-24; Hopper's e4m3 MMA keeps fewer mantissa bits in its internal sums, and
    on an H100 the observed error was 2^-11.3 at K = 768.  The bound, 2^-9, is the f16 output's own rounding (2^-11) with room for a
    longer K."""
    rng = np.random.default_rng(K)
    M, N = 1000, 512
    A = fr.e4m3_bits(rng.standard_normal((M, K)) * 40)
    W = fr.e4m3_bits(rng.standard_normal((N, K)) * 40)
    sa = rng.uniform(0.01, 0.02, M).astype(np.float32)
    sw = np.float32(0.003)
    bias = np.zeros(N, np.float32)
    out = eng.test_gemm_fp8(M, N, K, eng.EPI_BIAS_F16_HILO, A, sa, W, sw, bias)
    a, w = fr.e4m3_value(A).astype(np.float64), fr.e4m3_value(W).astype(np.float64)
    s = (sa.astype(np.float32) * sw).astype(np.float64)[:, None]  # the kernel rounds sa * sw to f32
    ref = (a @ w.T) * s
    mag = (np.abs(a) @ np.abs(w).T) * s
    err = (np.abs(out - ref) / mag).max()
    print(f"K = {K}: max |GPU - f64| / sum|a w| = {err:.3e} (2^{np.log2(err):.1f})")
    assert err <= 2.0 ** -9


# ---- LayerNorm -> e4m3 ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,D", [(1, 768), (7, 768), (8, 768), (9, 768), (591, 768), (1154, 1024), (4097, 128), (34, 128), (50, 192), (2, 384),
                                    (591, 256), (591, 384), (57, 512), (4097, 640), (300, 896), (9, 1536), (33, 2048)])
def test_layernorm_e4m3_matches_the_emulation(rows, D):
    """Both kernels (bulk-copy for D % 128 == 0 and >= 8 rows, row-per-warp otherwise), the row counts of
    test_layernorm_matches_the_restatement.  The kernel's f32 LayerNorm and the restatement's differ in the last bits, so a value near an
    e4m3 rounding boundary may land one step away, and the row scale a few f32 ulps away."""
    rng = np.random.default_rng(rows * 131 + D)
    x = (rng.standard_normal((rows, D)) * rng.uniform(0.5, 4.0, (rows, 1)) + rng.uniform(-1, 1, (rows, 1))).astype(np.float32)
    w = rng.uniform(0.5, 1.5, D).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, D).astype(np.float32)
    q, sa = eng.test_layernorm_fp8(x, w, b)
    q_ref, sa_ref = fr.quantize_rows(rs.layernorm(x, w, b))
    assert np.isfinite(sa).all() and (sa > 0).all()
    assert (np.abs(sa - sa_ref) <= 4 * np.spacing(sa_ref)).all()
    v, v_ref = fr.e4m3_value(q) * sa[:, None], fr.e4m3_value(q_ref) * sa_ref[:, None]
    # one e4m3 step at the reference code: 2^(e - 3) in binade e, 2^-9 among the subnormals
    step = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(fr.e4m3_value(q_ref)), 2.0 ** -6))) - 3)
    assert (np.abs(v - v_ref) <= 1.01 * step * sa_ref[:, None]).all()
    assert (q == q_ref).mean() > 0.995


def test_layernorm_e4m3_zero_row_gets_scale_one():
    x = np.zeros((16, 256), np.float32)
    q, sa = eng.test_layernorm_fp8(x, np.ones(256, np.float32), np.zeros(256, np.float32))
    assert (sa == 1).all() and not q.any()


# ---- end to end ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg,ftype", [("micro", "f16"), ("tiny", "f16"), ("tiny", "q8_0"), ("base", "f16")])
def test_logits_match_the_emulation(cfg, ftype):
    g = np.load(os.path.join(GOLD, f"{cfg}_{ftype}.npz"))
    path = model_path(cfg, ftype)
    vf = gf.read(path)
    imgs = gf.synthetic_images(int(g["n_images"]), vf.img_size, seed=int(g["image_seed"]))
    m = eng.vit_model_load(path, 0, 8, fp8=True)
    assert m.fp8
    probs, idx, val, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    m.close()
    emu = Emulation(vf).forward(imgs)
    d = fr.rel_dist(logits, emu)
    print(f"{cfg} {ftype}: GPU vs emulation {np.round(d, 4)}, GPU vs golden {np.round(fr.rel_dist(logits, g['logits']), 4)}")
    assert d.max() <= E2E_TOL
    L = g["logits"]
    top2 = np.sort(L, axis=1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 2 * E2E_TOL * np.abs(L).max(axis=1)
    assert (logits.argmax(1) == L.argmax(1))[clear].all()
    assert np.array_equal(val, np.take_along_axis(probs, idx.astype(np.int64), 1))


def test_taps_are_the_dequantised_layernorm_rows():
    path = model_path("micro", "f16")
    vf = gf.read(path)
    imgs = gf.synthetic_images(2, vf.img_size, seed=7)
    m = eng.vit_model_load(path, 0, 4, fp8=True)
    _, _, taps = eng.vit_predict_debug(m, imgs, 0, taps=("embed", "ln1", "x1", "ln2"))
    m.close()
    D = vf.hidden_size
    t = vf.tensors
    for name, x, wn in (("ln1", taps["embed"], "norm1"), ("ln2", taps["x1"], "norm2")):
        y = rs.layernorm(x.reshape(-1, D), np.asarray(t[f"blocks.0.{wn}.weight"], np.float32), np.asarray(t[f"blocks.0.{wn}.bias"], np.float32))
        q, sa = fr.quantize_rows(y)
        want = fr.e4m3_value(q) * sa[:, None]
        got = taps[name].reshape(-1, D)
        # the same e4m3 code on nearly every element; the row scale may sit a few f32 ulps from the emulation's (the kernel's f32 LayerNorm
        # against the restatement's), which moves every product of the row by as much
        assert (np.abs(got - want) <= 5e-7 * np.abs(want)).mean() > 0.99
        # where the f32 LayerNorms differ in the last bit a code may move one e4m3 step, at most 1/8 of the largest value
        assert np.abs(got - want).max() <= np.abs(want).max() / 8


# ---- every entry point ---------------------------------------------------------------------------------------------------------
def test_every_entry_point_on_an_fp8_engine():
    path = model_path("tiny", "f16")
    before = eng.vit_model_load(path, 0, 48)
    imgs = gf.synthetic_images(48, before.img_size, seed=3)
    p0, i0, v0, l0 = eng.vit_predict(before, imgs[:5], 5, want_logits=True)
    before.close()

    m = eng.vit_model_load(path, 0, 48, fp8=True)
    assert m.fp8
    # host, eager (48 x 197 tokens is past the graph cache) and graphed (1 and 3 images): the same rows
    p, i, v, l = eng.vit_predict(m, imgs, 5, want_logits=True)
    assert m.last_launch_count() == 3 + 7 * 12 + 3
    for sl in (slice(0, 1), slice(3, 6), slice(47, 48), slice(0, 1)):
        ps, is_, vs, ls = eng.vit_predict(m, imgs[sl], 5, want_logits=True)
        assert np.array_equal(ls, l[sl]) and np.array_equal(ps, p[sl]) and np.array_equal(is_, i[sl])
    # device pointers
    import torch
    d_img = torch.from_numpy(imgs[:4]).cuda()
    d_probs = torch.empty((4, m.num_classes), dtype=torch.float32, device="cuda")
    d_logits = torch.empty_like(d_probs)
    torch.cuda.synchronize()
    assert eng.lib().vitb200_forward_device(m.handle, d_img.data_ptr(), 4, d_probs.data_ptr(), d_logits.data_ptr(), None, None, 0, None) == 0
    assert eng.lib().vitb200_sync(m.handle) == 0
    torch.cuda.synchronize()
    assert np.array_equal(d_logits.cpu().numpy(), l[:4])
    # async: two batches in flight
    pa = np.empty((3, m.num_classes), np.float32)
    pb = np.empty((3, m.num_classes), np.float32)
    L = eng.lib()
    assert L.vitb200_forward_async(m.handle, np.ascontiguousarray(imgs[0:3]).ctypes.data, 3, pa.ctypes.data, None, None, None, 0) == 0
    keep = np.ascontiguousarray(imgs[3:6])
    assert L.vitb200_forward_async(m.handle, keep.ctypes.data, 3, pb.ctypes.data, None, None, None, 0) == 0
    assert L.vitb200_sync(m.handle) == 0
    assert np.array_equal(pa, p[0:3]) and np.array_equal(pb, p[3:6])
    # sharded over one engine
    ps, is_, vs = eng.vit_predict_sharded([m], imgs[:6])
    assert np.array_equal(ps, p[:6])
    # features: the residual stream and the pre-logits rows
    tok, pre = eng.vit_features(m, imgs[:2], prelogits=True)
    assert tok.shape == (2, m.n_tokens, m.hidden_size) and np.isfinite(tok).all()
    assert np.array_equal(pre[:, 0], tok[:, 0])
    # u8: the GPU preprocess feeds the same FP8 forward
    rng = np.random.default_rng(9)
    u8 = [rng.integers(0, 256, size=(300, 260, 3), dtype=np.uint8) for _ in range(3)]
    f32, pu, iu, vu, lu = eng.vit_image_preprocess_predict(m, u8)
    pf, _, _, lf = eng.vit_predict(m, f32, 5, want_logits=True)
    assert np.array_equal(lu, lf)
    tu, _ = eng.vit_features_u8(m, u8)
    assert tu.shape[0] == 3 and np.isfinite(tu).all()
    # FP8 outputs differ from f16 ones, within the end-to-end tolerance of the recipe
    assert not np.array_equal(l[:5], l0)
    assert fr.rel_dist(l[:5], l0).max() <= 0.2
    m.close()

    # a default engine built after the FP8 one computes exactly what one built before it did
    after = eng.vit_model_load(path, 0, 48)
    p1, i1, v1, l1 = eng.vit_predict(after, imgs[:5], 5, want_logits=True)
    assert not after.fp8
    assert np.array_equal(l1, l0) and np.array_equal(p1, p0) and np.array_equal(i1, i0)
    after.close()


def test_launch_count_micro_and_base():
    for cfg, n in (("micro", 5), ("base", 3)):
        imgs = gf.synthetic_images(n, gf.CONFIGS[cfg][4], seed=12)
        m = eng.vit_model_load(model_path(cfg, "f16"), 0, 8, fp8=True)
        eng.vit_predict(m, imgs, 5)
        assert m.last_launch_count() == 3 + 7 * gf.CONFIGS[cfg][1] + 3
        m.close()


def test_from_tensors_equals_from_file():
    path = model_path("micro", "f16")
    vf = gf.read(path)
    imgs = gf.synthetic_images(3, vf.img_size, seed=4)
    a = eng.vit_model_load(path, 0, 4, fp8=True)
    b = eng.vit_model_from_tensors(vf, 0, 4, fp8=True)
    assert b.fp8
    la = eng.vit_predict(a, imgs, 5, want_logits=True)[3]
    lb = eng.vit_predict(b, imgs, 5, want_logits=True)[3]
    assert np.array_equal(la, lb)
    a.close()
    b.close()


def test_vitstr_recognition_on_an_fp8_engine():
    g = np.load(os.path.join(GOLD, "vitstr_micro_f16.npz"))
    path = model_path("vitstr_micro", "f16")
    vf = gf.read(path)
    m = eng.vit_model_load(path, 0, 8, head_tokens=25, fp8=True)
    assert m.fp8 and m.head_tokens == 25
    imgs = gf.synthetic_gray_images(int(g["n_images"]), vf.img_size, seed=int(g["image_seed"]))
    probs, idx, val, logits = eng.vit_predict(m, imgs, 1, want_logits=True)
    emu = Emulation(vf, head_tokens=25).forward(imgs)
    assert fr.rel_dist(logits, emu).max() <= E2E_TOL
    rng = np.random.default_rng(2)
    u8 = [rng.integers(0, 256, size=(32, 100, 3), dtype=np.uint8) for _ in range(4)]
    texts, scores, chars, lengths, pr = eng.vitstr_recognize_u8(m, u8, probs=True)
    gray = eng.vitstr_preprocess_u8(m, u8)
    p2 = eng.vit_predict(m, gray, 1)[0]
    assert np.array_equal(pr, p2)
    am = p2[:, 1:].argmax(axis=2)
    for b in range(4):
        n = int(lengths[b])
        assert np.array_equal(chars[b, :n], am[b, :n])
        assert n == 24 or am[b, n] == 1
    m.close()
