"""The persistent wgmma GEMM's tile schedule, checked element by element.

The GEMM runs a persistent grid of two-CTA clusters; each cluster walks pairs of column tiles (one per CTA, sharing the A tile
through multicast), and each CTA hands its tiles alternately to two MMA warpgroups, with one operand ring whose slots and barrier
phases carry across tiles.  A tile sent to the wrong CTA or warpgroup, a barrier phase that slips at a tile boundary, or a staging
buffer reused too early corrupts whole tiles, so every element is compared exactly: A and W hold small integers, so every partial
sum, and the result, is an integer well inside f32's exact range.

The activation, LayerScale and SwiGLU epilogues (7 - 11) take W in quarter-integers instead, so that x = acc + bias, still exact in
f32, lands on fractional values near 0 where the activations bend.  Their outputs are checked as functions: the same x (or, for
SwiGLU, the same pair x1, x2) must give the same bits at every position, and that value must be within the rounding of the f16 result
of a float64 evaluation.  A tile written from another tile's accumulators, columns or bias breaks the first condition."""
import math

import numpy as np
import pytest
from scipy.special import ndtr

from tests.util import pkg
from tests.emulation import gelu_pytorch_tanh
from oracle import restatement as rs

eng = pkg.engine
pytestmark = pytest.mark.gpu

BM = BN = 128  # the GEMM's tile
ACTIVATIONS = (eng.EPI_BIAS_GELU_ERF_F16, eng.EPI_BIAS_QUICK_GELU_F16, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16)
NEW = ACTIVATIONS + (eng.EPI_BIAS_SCALE_RESID_F32, eng.EPI_SWIGLU)
TAIL_EVERY = 61  # every 61st bias column (of x1 for SwiGLU) is -1e4: the far left tail, in a different place in every tile


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def act64(x, epi):
    """The activation of epilogue 7, 8 or 10 in float64."""
    x = np.asarray(x, np.float64)
    if epi == eng.EPI_BIAS_GELU_ERF_F16:
        return x * ndtr(x)
    if epi == eng.EPI_BIAS_QUICK_GELU_F16:
        with np.errstate(over="ignore"):
            return x / (1.0 + np.exp(-1.702 * x))
    if epi == eng.EPI_BIAS_GELU_PYTORCH_TANH_F16:
        return gelu_pytorch_tanh(x)
    raise ValueError(epi)


def _distinct(q):
    """Dense ranks of the integers q and the sorted distinct values (bincount: np.unique sorts, too slow at full size)."""
    lo = int(q.min())
    present = np.bincount((q - lo).ravel()) > 0
    return (np.cumsum(present) - 1)[q - lo], np.flatnonzero(present) + lo


def function_of(out, key):
    """out with every element replaced by the value out takes at some position of the same integer key; and the distinct keys with
    those values.  Equal to out bit for bit exactly when out is a function of the key."""
    flat = key.ravel()
    per = np.zeros(int(flat.max()) + 1, out.dtype)
    per[flat] = out.ravel()
    seen = np.flatnonzero(np.bincount(flat))
    return per[flat].reshape(out.shape), seen, per[seen]


def check_activation(out, q, step, epi):
    """Epilogues 7, 8, 10 on exact pre-activations x = q step (q integer): out a function of x, within one f16 ulp of f16(act(x)) in
    float64 (so never NaN), and -0 wherever a negative x's activation rounds to zero in f16 (x < -10 for 7 and 10, x < -16 for 8; the
    bias takes some x to -1e4).  Returns the expected array (out itself when out is a function of x)."""
    lo = int(q.min())
    want, seen, vals = function_of(out, q - lo)
    xs = (seen + lo) * step
    ref16 = act64(xs, epi).astype(np.float16)
    err = np.abs(vals.astype(np.float64) - ref16.astype(np.float64))
    bad = ~(err <= np.spacing(np.abs(ref16)).astype(np.float64))
    assert not bad.any(), f"epilogue {epi}: x = {xs[bad][:5]} gives {vals[bad][:5]}, f16(act(x)) = {ref16[bad][:5]}"
    tail = (xs < 0) & (ref16 == 0)
    assert xs.min() < -1000 and (vals[tail] == 0).all() and np.signbit(vals[tail]).all(), f"epilogue {epi}: tail gives {vals[tail][:5]}"
    return want


def check_swiglu(out, q1, q2, step):
    """Epilogue 11 on exact x1 = q1 step, x2 = q2 step (q integer): out a function of the pair (x1, x2), within _silu_bound of float64
    with exact inputs, and 0 for x1 < -100 (e^-x1 overflows f32).  Returns the expected array, as check_activation does."""
    from tests.test_gpu_swiglu import _silu_bound  # here: that module imports test_gpu_fp8, which imports this one
    r1, u1 = _distinct(q1)
    r2, u2 = _distinct(q2)
    want, seen, vals = function_of(out, r1 * u2.size + r2)
    x1, x2 = u1[seen // u2.size] * step, u2[seen % u2.size] * step
    ref, tol = _silu_bound(x1, x2, 0, 0)
    assert np.abs(ref).max() < 65504, "operands too large: the products leave the f16 range"
    bad = ~(np.abs(vals - ref) <= tol)
    assert not bad.any(), f"SwiGLU: (x1, x2) = {list(zip(x1[bad][:5], x2[bad][:5]))} gives {vals[bad][:5]}, want {ref[bad][:5]}"
    tail = x1 < -100
    assert tail.any() and (vals[tail] == 0).all(), f"SwiGLU: x1 < -100 gives {vals[tail][:5]}"
    return want


def assert_same_bits(out, want):
    bad = out.view(np.uint32) != want.view(np.uint32)
    if bad.any():
        r, c = np.argwhere(bad)[0]
        tiles = sorted({(int(i) // BM, int(j) // BN) for i, j in np.argwhere(bad)[:100000]})
        raise AssertionError(f"{int(bad.sum())} of {bad.size} elements differ; first at row {r} col {c}: {out[r, c]} != {want[r, c]}; "
                             f"tiles (m, n) {tiles[:8]}{' ...' if len(tiles) > 8 else ''}")


def _check_new(M, N, K, epi, rng):
    """Epilogues 7 - 11.  A: integers in [-2, 2] (SwiGLU: sparse, at most ~64 per row, so that silu(x1) x2 stays inside the f16 range);
    W = W4 / 4 with W4 integers in [-8, 8]; bias: integers in [-8, 8] and -1e4 in every TAIL_EVERY-th column.  SwiGLU takes N = 2 F in
    HF's order and returns [M][F]."""
    F = N // 2
    A = rng.integers(-2, 3, size=(M, K), dtype=np.int8)
    if epi == eng.EPI_SWIGLU:
        A *= (rng.random((M, K)) < min(1.0, 64.0 / K)).astype(np.int8)
    W4 = rng.integers(-8, 9, size=(N, K), dtype=np.int8)
    bias = rng.integers(-8, 9, size=N).astype(np.float32)
    bias[:F if epi == eng.EPI_SWIGLU else N:TAIL_EVERY] = -1e4
    A16, W16 = A.astype(np.float16), (W4.astype(np.float32) / 4).astype(np.float16)
    if epi == eng.EPI_BIAS_SCALE_RESID_F32:
        gamma = np.exp(rng.uniform(np.log(1e-6), np.log(10.0), N)).astype(np.float32)
        resid = (rng.standard_normal((M, N)) * 16).astype(np.float32)
        out = eng.test_gemm_layer_scale(M, N, K, A16, W16, bias, gamma, resid)
    else:
        out = eng.test_gemm(M, N, K, epi, A16, W16, bias)
    # q = 4 x = A W4^T + 4 bias: |partial sums| <= 16 K < 2^24, so the f32 BLAS is exact integer arithmetic in any order
    q = (A.astype(np.float32) @ W4.astype(np.float32).T).astype(np.int64)
    for r in (0, M // 2, M - 1):
        assert np.array_equal(q[r], A[r].astype(np.int64) @ W4.astype(np.int64).T)
    q += (4 * bias).astype(np.int64)
    if epi == eng.EPI_BIAS_SCALE_RESID_F32:
        # the kernel rounds x * gamma, then the sum (__fmul_rn, __fadd_rn): numpy's f32 arithmetic is the same two IEEE roundings
        want = (q.astype(np.float32) * np.float32(0.25)) * gamma + resid
    elif epi == eng.EPI_SWIGLU:
        assert out.shape == (M, F)
        want = check_swiglu(out, q[:, :F], q[:, F:], 0.25)
    else:
        want = check_activation(out, q, 0.25, epi)
    assert_same_bits(out, want)


def _check(M, N, K, epi, seed):
    rng = np.random.default_rng(seed)
    if epi in NEW:
        return _check_new(M, N, K, epi, rng)
    A = rng.integers(-2, 3, size=(M, K)).astype(np.float16)
    W = rng.integers(-2, 3, size=(N, K)).astype(np.float16)
    bias = rng.integers(-8, 9, size=N).astype(np.float32)
    resid = rng.integers(-64, 65, size=(M, N)).astype(np.float32) if epi == eng.EPI_BIAS_RESID_F32 else None
    out = eng.test_gemm(M, N, K, epi, A, W, bias, resid)  # the residual epilogue runs in place: resid aliases out
    # |partial sums| <= 4 K < 2^24: the f32 product is exact integer arithmetic, whatever order the BLAS sums in
    acc = (A.astype(np.float32) @ W.astype(np.float32).T).astype(np.int64)
    for r in (0, M // 2, M - 1):
        assert np.array_equal(acc[r], A[r].astype(np.int64) @ W.astype(np.int64).T)
    x = (acc + bias.astype(np.int64)).astype(np.float32)
    if epi == eng.EPI_BIAS_RESID_F32:
        want = x + resid
    elif epi == eng.EPI_BIAS_F32:
        want = x
    elif epi == eng.EPI_BIAS_F16_HILO:
        # |x| < 2048 is exact in f16: hi = x and lo = 0, and test_gemm returns hi + lo
        assert np.abs(x).max() < 2048
        want = x
    elif epi == eng.EPI_BIAS_F16:
        want = x.astype(np.float16).astype(np.float32)
    elif epi == eng.EPI_BIAS_GELU_F16:
        # The kernel evaluates GELU in f32 (gemm_wgmma.cuh) and rounds to f16 one ulp away from the reference table on a few
        # inputs, so each output must be a function of its pre-activation -- the same at every position -- that is the table's
        # value to within one f16 ulp.  A misplaced tile breaks the first condition.
        x16 = x.astype(np.float16).astype(np.float32)
        xi = x16.astype(np.int64).ravel() - int(x16.min())  # integers: f16 holds them exactly below 2048
        assert np.abs(x).max() < 2048
        per_value = np.zeros(int(xi.max()) + 1, np.float32)
        per_value[xi] = out.ravel()
        want = per_value[xi].reshape(out.shape)
        seen = np.flatnonzero(np.bincount(xi))
        table = rs.gelu_table((seen + int(x16.min())).astype(np.float32))
        ulp = np.maximum(np.abs(table), 2.0 ** -14) * 2.0 ** -10
        assert (np.abs(per_value[seen] - table) <= ulp).all()
    else:
        raise ValueError(epi)
    bad = out != want
    if bad.any():
        r, c = np.argwhere(bad)[0]
        tiles = sorted({(int(i) // BM, int(j) // BN) for i, j in np.argwhere(bad)[:100000]})
        raise AssertionError(f"{int(bad.sum())} of {bad.size} elements differ; first at row {r} col {c}: {out[r, c]} != {want[r, c]}; "
                             f"tiles (m, n) {tiles[:8]}{' ...' if len(tiles) > 8 else ''}")


@pytest.mark.parametrize("epi", [eng.EPI_BIAS_F32, eng.EPI_BIAS_F16] + list(NEW))
def test_fewer_tiles_than_sms(epi):
    """The head shape: 2 x 8 tiles, each CTA has one tile and its second warpgroup none; the last column tile is partial.  SwiGLU with
    F = 344: 2 x 6 tiles, the last group of 64 hidden units partial."""
    _check(256, 2 * 344 if epi == eng.EPI_SWIGLU else 1000, 768, epi, seed=1)


_GRID_NEW = [(K, e) for e in NEW for K in (192, 320, 2048, 3072)]

# (N, K, epilogue) with K % 64 != 0: the last k-block of every tile is partly past K, and TMA zero-fills that part of both operands.  The
# reductions the engine runs: D at head dims 72 and 80 with an odd head count (72, 80, 240, ...), the So400m micro towers (144), MLP
# widths read from the weights as fc2's K (344, 464, 2736, So400m's 4304), down to a single partial k-block (8, 24, 56); 2736 and 4304
# run the 6-stage ring.  Every epilogue family at least once.
K_TAILS = [(384, 8, eng.EPI_BIAS_F16), (384, 24, eng.EPI_BIAS_RESID_F32), (384, 56, eng.EPI_BIAS_F32), (384, 72, eng.EPI_BIAS_F16_HILO),
           (384, 80, eng.EPI_BIAS_GELU_F16), (384, 144, eng.EPI_BIAS_GELU_ERF_F16), (384, 240, eng.EPI_BIAS_QUICK_GELU_F16),
           (384, 344, eng.EPI_BIAS_SCALE_RESID_F32), (384, 464, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16), (2 * 2736, 72, eng.EPI_SWIGLU),
           (384, 2736, eng.EPI_BIAS_F16), (384, 2736, eng.EPI_BIAS_SCALE_RESID_F32), (2 * 2736, 2736, eng.EPI_SWIGLU),
           (384, 4304, eng.EPI_BIAS_RESID_F32), (384, 4304, eng.EPI_BIAS_F16_HILO), (384, 4304, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16)]


@pytest.mark.parametrize("per_cluster,extra", [(4, 0), (4, 1), (4, -1), (3, 0), (3, 1)])
@pytest.mark.parametrize("K,epi", [(192, eng.EPI_BIAS_F16), (64, eng.EPI_BIAS_RESID_F32), (320, eng.EPI_BIAS_F16_HILO),
                                   (2048, eng.EPI_BIAS_F16_HILO), (80, eng.EPI_BIAS_F16_HILO), (344, eng.EPI_BIAS_F16),
                                   (4304, eng.EPI_BIAS_RESID_F32)] + _GRID_NEW)
def test_tile_counts_around_the_grid(per_cluster, extra, K, epi):
    """per_cluster x SMs / 2 tile pairs (+ extra).  The engine launches as many clusters as fit at once, which is SMs / 2 on an H100
    SXM; where fewer fit, these counts are still uneven shares of the grid, only not the exact boundaries named here.  With SMs / 2
    clusters: equal shares, one cluster with one more, one with one fewer; an odd share gives the first warpgroup one tile more than
    the second.  K = 64, 192, 320 are 1, 3 and 5 k-blocks against the 5-slot ring, so tiles start at every slot and phase; K = 2048
    (32 k-blocks) and 3072 run the 6-slot ring with the smaller staging buffer (and LayerScale's gamma staged per pass).  K = 80, 344
    and 4304 (2, 6 and 68 k-blocks) end each tile's reduction in a k-block TMA zero-fills past K, on both rings.  SwiGLU with F = 128:
    one pair per row band, as for the other epilogues."""
    pairs = per_cluster * (_sms() // 2) + extra
    _check(pairs * BM, 2 * BN, K, epi, seed=pairs + K)


@pytest.mark.parametrize("N,K,epi", [(128, 448, eng.EPI_BIAS_F16), (128, 448, eng.EPI_BIAS_RESID_F32), (384, 448, eng.EPI_BIAS_F16_HILO),
                                     (384, 448, eng.EPI_BIAS_F32), (384, 448, eng.EPI_BIAS_GELU_F16), (384, 2048, eng.EPI_BIAS_RESID_F32),
                                     (384, 448, eng.EPI_BIAS_GELU_ERF_F16), (384, 2048, eng.EPI_BIAS_QUICK_GELU_F16),
                                     (384, 448, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16), (128, 448, eng.EPI_BIAS_SCALE_RESID_F32),
                                     (384, 3072, eng.EPI_BIAS_SCALE_RESID_F32), (2 * 2736, 448, eng.EPI_SWIGLU),
                                     (2 * 2736, 2048, eng.EPI_SWIGLU)] + K_TAILS)
def test_odd_column_tile_count(N, K, epi):
    """An odd number of column tiles: the second CTA of the last pair computes a tile past N, stores nothing, and still releases its
    share of the ring it shares with the first.  SwiGLU with F = 2736: 43 column tiles.  K_TAILS: reductions whose last k-block is
    partly zero-filled."""
    _check(197 * 7, N, K, epi, seed=N + K + epi)


@pytest.mark.parametrize("N,epi", [(768, eng.EPI_BIAS_RESID_F32), (3072, eng.EPI_BIAS_GELU_F16), (2304, eng.EPI_BIAS_F16_HILO),
                                   (3072, eng.EPI_BIAS_GELU_ERF_F16), (3072, eng.EPI_BIAS_QUICK_GELU_F16),
                                   (3072, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16), (768, eng.EPI_BIAS_SCALE_RESID_F32),
                                   (2 * 344, eng.EPI_SWIGLU)])
def test_m_tail(N, epi):
    """M = 197 x 255 ends inside a tile's second 64-row half: those rows are computed from zero fill and never stored."""
    _check(197 * 255, N, 768, epi, seed=N + epi)


@pytest.mark.parametrize("epi", NEW)
@pytest.mark.parametrize("K", [768, 3072])
def test_warpgroups_take_different_column_tiles(epi, K):
    """Cluster c takes pairs c, c + clusters, ... and its warpgroups alternate between them, so when the pairs per row band divide the
    cluster count (1 for N = 256, 3 for N = 768 on 66 clusters) each CTA keeps one column tile and both warpgroups see the same
    columns: a bias or gamma read from the other warpgroup's shared-memory slot still looks right.  Here the pair count is coprime to
    the cluster count, so the two warpgroups of a CTA run different column tiles; M = 197 x 63 ends in a tile's second row half.
    K = 768 runs the 5-stage ring, 3072 the 6-stage one (LayerScale's gamma staged per pass)."""
    clusters = _sms() // 2
    n_pairs = next(n for n in (5, 7, 11, 13) if math.gcd(n, clusters) == 1)
    N = 2 * BN * n_pairs  # SwiGLU: F = N / 2 is a multiple of 64, so the interleaved GEMM has N columns too
    _check(197 * 63, N, K, epi, seed=N + K + epi)


@pytest.mark.parametrize("N,K,epi", [(768, 768, eng.EPI_BIAS_RESID_F32), (2304, 768, eng.EPI_BIAS_F16_HILO), (2304, 768, eng.EPI_BIAS_F16),
                                     (3072, 768, eng.EPI_BIAS_GELU_F16), (768, 3072, eng.EPI_BIAS_RESID_F32),
                                     (3072, 768, eng.EPI_BIAS_GELU_ERF_F16), (3072, 768, eng.EPI_BIAS_QUICK_GELU_F16),
                                     (3072, 768, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16), (768, 768, eng.EPI_BIAS_SCALE_RESID_F32),
                                     (768, 3072, eng.EPI_BIAS_SCALE_RESID_F32), (2 * 4096, 1536, eng.EPI_SWIGLU)])
def test_full_size(N, K, epi):
    """The ViT-B/16 block GEMMs at batch 256 (M = 256 x 197): proj, qkv (split and plain), fc1 (tanh GELU with the f16 table, erf,
    QuickGELU and PyTorch's tanh GELU) and fc2, the residual ones in place; DINOv2 B/14 with 4 registers (261 tokens) at batch 256: the
    LayerScale proj and fc2; ViT-g's SwiGLU fc1 (F = 4096) at batch 64."""
    M = {eng.EPI_BIAS_SCALE_RESID_F32: 256 * 261, eng.EPI_SWIGLU: 64 * 261}.get(epi, 256 * 197)
    _check(M, N, K, epi, seed=N * 7 + K + epi)


# (M, N, K, epilogue): the block GEMMs of the towers with widths that are not multiples of 128, for 3 images
TOWER_LAYERS = [
    (729 * 3, 3456, 1152, eng.EPI_BIAS_F16_HILO),                # SigLIP So400m at 384 px: qkv (27 column tiles)
    (729 * 3, 4304, 1152, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16),   # fc1: the last column tile holds 80 columns
    (729 * 3, 1152, 4304, eng.EPI_BIAS_RESID_F32),               # fc2: K = 4304, a 16-column last k-block on the 6-stage ring
    (257 * 3, 3840, 1280, eng.EPI_BIAS_F16_HILO),                # ViT-H/14 at 224 px: qkv (30 column tiles)
    (257 * 3, 5120, 1280, eng.EPI_BIAS_GELU_ERF_F16),            # fc1, erf GELU
    (257 * 3, 1280, 5120, eng.EPI_BIAS_RESID_F32),               # fc2
]


@pytest.mark.parametrize("M,N,K,epi", TOWER_LAYERS)
def test_tower_layer_shapes(M, N, K, epi):
    """So400m and ViT-H/14 layers once each; M = 3 x 729 and 3 x 257 end 11 and 3 rows into their last row tile."""
    _check(M, N, K, epi, seed=M + N + K + epi)
