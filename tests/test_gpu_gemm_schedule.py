"""The persistent wgmma GEMM's tile schedule, checked element by element.

The GEMM runs a persistent grid of two-CTA clusters; each cluster walks pairs of column tiles (one per CTA, sharing the A tile
through multicast), and each CTA hands its tiles alternately to two MMA warpgroups, with one operand ring whose slots and barrier
phases carry across tiles.  A tile sent to the wrong CTA or warpgroup, a barrier phase that slips at a tile boundary, or a staging
buffer reused too early corrupts whole tiles, so every element is compared exactly: A and W hold small integers, so every partial
sum, and the result, is an integer well inside f32's exact range."""
import numpy as np
import pytest

from tests.util import pkg
from oracle import restatement as rs

eng = pkg.engine
pytestmark = pytest.mark.gpu

BM = BN = 128  # the GEMM's tile


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check(M, N, K, epi, seed):
    rng = np.random.default_rng(seed)
    A = rng.integers(-2, 3, size=(M, K)).astype(np.float16)
    W = rng.integers(-2, 3, size=(N, K)).astype(np.float16)
    bias = rng.integers(-8, 9, size=N).astype(np.float32)
    resid = rng.integers(-64, 65, size=(M, N)).astype(np.float32) if epi == 2 else None
    out = eng.test_gemm(M, N, K, epi, A, W, bias, resid)  # the residual epilogue runs in place: resid aliases out
    # |partial sums| <= 4 K < 2^24: the f32 product is exact integer arithmetic, whatever order the BLAS sums in
    acc = (A.astype(np.float32) @ W.astype(np.float32).T).astype(np.int64)
    for r in (0, M // 2, M - 1):
        assert np.array_equal(acc[r], A[r].astype(np.int64) @ W.astype(np.int64).T)
    x = (acc + bias.astype(np.int64)).astype(np.float32)
    if epi == 2:
        want = x + resid
    elif epi == 4:
        want = x
    elif epi == 6:
        # |x| < 2048 is exact in f16: hi = x and lo = 0, and test_gemm returns hi + lo
        assert np.abs(x).max() < 2048
        want = x
    elif epi == 0:
        want = x.astype(np.float16).astype(np.float32)
    elif epi == 1:
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


@pytest.mark.parametrize("epi", [4, 0])
def test_fewer_tiles_than_sms(epi):
    """The head shape: 2 x 8 tiles, each CTA has one tile and its second warpgroup none; the last column tile is partial."""
    _check(256, 1000, 768, epi, seed=1)


@pytest.mark.parametrize("per_cluster,extra", [(4, 0), (4, 1), (4, -1), (3, 0), (3, 1)])
@pytest.mark.parametrize("K,epi", [(192, 0), (64, 2), (320, 6), (2048, 6)])
def test_tile_counts_around_the_grid(per_cluster, extra, K, epi):
    """per_cluster x SMs / 2 tile pairs (+ extra).  The engine launches as many clusters as fit at once, which is SMs / 2 on an H100
    SXM; where fewer fit, these counts are still uneven shares of the grid, only not the exact boundaries named here.  With SMs / 2
    clusters: equal shares, one cluster with one more, one with one fewer; an odd share gives the first warpgroup one tile more than
    the second.  K = 64, 192, 320 are 1, 3 and 5 k-blocks against the 5-slot ring, so tiles start at every slot and phase; K = 2048
    (32 k-blocks) runs the 6-slot ring with the smaller staging buffer."""
    pairs = per_cluster * (_sms() // 2) + extra
    _check(pairs * BM, 2 * BN, K, epi, seed=pairs + K)


@pytest.mark.parametrize("N,K,epi", [(128, 448, 0), (128, 448, 2), (384, 448, 6), (384, 448, 4), (384, 448, 1), (384, 2048, 2)])
def test_odd_column_tile_count(N, K, epi):
    """An odd number of column tiles: the second CTA of the last pair computes a tile past N, stores nothing, and still releases its
    share of the ring it shares with the first."""
    _check(197 * 7, N, K, epi, seed=N + K + epi)


@pytest.mark.parametrize("N,epi", [(768, 2), (3072, 1), (2304, 6)])
def test_m_tail(N, epi):
    """M = 197 x 255 ends inside a tile's second 64-row half: those rows are computed from zero fill and never stored."""
    _check(197 * 255, N, 768, epi, seed=N + epi)


@pytest.mark.parametrize("N,K,epi", [(768, 768, 2), (2304, 768, 6), (2304, 768, 0), (3072, 768, 1), (768, 3072, 2)])
def test_full_size(N, K, epi):
    """The ViT-B/16 block GEMMs at batch 256 (M = 256 x 197): proj, qkv (split and plain), fc1 and fc2, the residual ones in place."""
    _check(256 * 197, N, K, epi, seed=N * 7 + K + epi)
