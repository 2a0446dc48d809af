"""The wgmma GEMM's head-major store, checked bit by bit.

At head dim 64 the qkv GEMM and the attention-pooling head's k | v GEMM write their output as planes [N / 64][plane_rows][64] with
plane_rows = max_batch x tokens, one plane per head's q, k or v slice, through a 3-D TMA store map; the split-precision form writes the
lo planes through a second map.  A call with fewer images than max_batch has M < plane_rows, and the rows M .. plane_rows - 1 of every
plane must stay untouched.  The hook fills both outputs with 0xFFFF first, so a row past M that is stored, a plane index off by one or
a lo box stored into a hi plane shows up here.

Operands are small integers (f16, or e4m3 with power-of-two scales as tests/test_gpu_fp8.py takes them), so x = acc + bias is exact in
f32.  The bias has an odd multiple of 2^-8 in every column, so x has more significant bits than f16 holds wherever |x| >= 8, and there
lo = f16(x - hi) is non-zero: a lo plane swapped with another or with its hi plane cannot pass for zeros."""
import math

import numpy as np
import pytest

from tests.util import pkg
from tests import fp8_reference as fr

eng = pkg.engine
pytestmark = pytest.mark.gpu

SENTINEL = 0xFFFF
EPIS = [eng.EPI_BIAS_F16, eng.EPI_BIAS_F16_HILO]


def _operands(M, N, K, e4m3, rng):
    """A, W, the A scales (e4m3) or None, the W scale, bias, and x [M][N] float32 = exactly what the kernel's epilogue starts from."""
    bias = ((2 * rng.integers(-4096, 4096, size=N) + 1) / 256).astype(np.float32)  # |bias| < 32, an odd multiple of 2^-8
    if not e4m3:
        A = rng.integers(-2, 3, size=(M, K))
        W = rng.integers(-2, 3, size=(N, K))
        acc = A.astype(np.float64) @ W.astype(np.float64).T  # integers, |partial sums| <= 4 K < 2^24: exact in the kernel's f32 too
        return A.astype(np.float16), W.astype(np.float16), None, 1.0, bias, (acc + bias).astype(np.float32)
    # as test_gpu_fp8._check_exact: sum_k |a| |w| < 2^11 on every row, whatever width Hopper's e4m3 MMA keeps in its sums
    A = rng.integers(-2, 3, size=(M, K)) * (rng.random((M, K)) < min(1.0, 96.0 / K))
    W = rng.integers(-4, 5, size=(N, K))
    assert (np.abs(A).sum(axis=1) * 4 < 2 ** 11).all()
    sa = (2.0 ** rng.integers(-1, 2, size=M)).astype(np.float32)
    sw = np.float32(0.25)
    acc = A.astype(np.float64) @ W.astype(np.float64).T
    x = (acc * (sa[:, None].astype(np.float64) * sw) + bias).astype(np.float32)  # multiples of 2^-8 below 2^11: exact
    return fr.e4m3_bits(A), fr.e4m3_bits(W), sa, sw, bias, x


def _planes(rows, plane_rows):
    """[M][N] uint16 -> [N / 64][plane_rows][64], rows past M the sentinel."""
    M, N = rows.shape
    out = np.full((N // 64, plane_rows, 64), SENTINEL, np.uint16)
    out[:, :M] = rows.reshape(M, N // 64, 64).transpose(1, 0, 2)
    return out


def _assert_planes(got, want, what):
    bad = got != want
    if bad.any():
        p, r, c = np.argwhere(bad)[0]
        planes = sorted({int(i) for i in np.argwhere(bad)[:100000, 0]})
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} halves differ; first in plane {p}, row {r}, column {c}: "
                             f"{got[p, r, c]:#06x} != {want[p, r, c]:#06x}; planes {planes[:8]}{' ...' if len(planes) > 8 else ''}")


def _check(M, N, K, plane_rows, epi, e4m3, seed):
    rng = np.random.default_rng(seed)
    A, W, sa, sw, bias, x = _operands(M, N, K, e4m3, rng)
    hi, lo = eng.test_gemm_planes(M, N, K, epi, A, W, bias, plane_rows, a_scale=sa, w_scale=sw)
    assert hi.shape == (N // 64, plane_rows, 64) and (lo is None) == (epi == eng.EPI_BIAS_F16)
    hi_want = x.astype(np.float16)  # round to nearest even, as __floats2half2_rn
    _assert_planes(hi, _planes(hi_want.view(np.uint16), plane_rows), "hi")
    if lo is None:
        return
    lo_want = (x - hi_want.astype(np.float32)).astype(np.float16)  # x - hi is exact in f32
    assert np.array_equal(hi_want.astype(np.float32) + lo_want.astype(np.float32), x)
    # most elements carry a non-zero lo (|x| >= 8): a lo plane written with zeros, or not at all, cannot pass
    assert (lo_want != 0).mean() > 0.5, (lo_want != 0).mean()
    _assert_planes(lo, _planes(lo_want.view(np.uint16), plane_rows), "lo")


def _clusters():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count // 2


# (M, N, K, plane_rows): qkv, N = 3 D, K = D; M = B x tokens for a batch of B out of max_batch = plane_rows / tokens
QKV = [
    (197 * 3, 192, 64, 197 * 4),      # D = 64: one k-block; 2 column tiles, the second half past N
    (197 * 3, 576, 192, 197 * 8),     # ViT-Ti (D = 192): 5 column tiles, the last pair's second tile past N
    (197 * 3, 2304, 768, 197 * 3),    # ViT-B: a full batch, plane_rows == M (= 4 x 128 + 79 rows)
    (257 * 2, 3072, 1024, 257 * 4),   # ViT-L/14
    (261 * 2, 6144, 2048, 261 * 3),   # D = 2048: the 6-stage ring, whose hi + lo passes are 64 columns wide
    (50 * 5, 1344, 448, 50 * 7),      # 7 heads: 11 column tiles
]
# the attention-pooling head's k | v GEMM: N = 2 D, M = B x patch rows
KV = [
    (196 * 3, 1536, 768, 196 * 4),
    (576 * 1, 2048, 1024, 576 * 2),   # SigLIP-L/16 at 384 px
]


@pytest.mark.parametrize("e4m3", [False, True], ids=["f16", "e4m3"])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("M,N,K,plane_rows", QKV)
def test_qkv_planes(M, N, K, plane_rows, epi, e4m3):
    _check(M, N, K, plane_rows, epi, e4m3, seed=M + N + K + epi)


@pytest.mark.parametrize("e4m3", [False, True], ids=["f16", "e4m3"])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("M,N,K,plane_rows", KV)
def test_pool_kv_planes(M, N, K, plane_rows, epi, e4m3):
    _check(M, N, K, plane_rows, epi, e4m3, seed=M + N + K + epi + 1)


@pytest.mark.parametrize("e4m3", [False, True], ids=["f16", "e4m3"])
@pytest.mark.parametrize("epi", EPIS)
def test_planes_with_an_odd_column_tile_count_coprime_to_the_clusters(epi, e4m3):
    """2 n - 1 column tiles, the last one 64 columns wide and the last pair's second CTA past N (computed, never stored), with n pairs
    per row band coprime to the cluster count: each cluster walks many row bands, and the two warpgroups of a CTA write different planes.
    M = 197 x 21 of plane_rows = 197 x 24 ends inside a tile's second 64-row half."""
    pairs = next(n for n in (5, 7, 11, 13) if math.gcd(n, _clusters()) == 1)
    N = (2 * pairs - 1) * 128 - 64
    _check(197 * 21, N, 320, 197 * 24, epi, e4m3, seed=N + epi)
