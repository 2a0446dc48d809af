"""GPU tests of individual kernels through the C ABI (vitb200_test_gemm) against numpy / the oracle's primitives."""
from typing import Callable, NamedTuple

import numpy as np
import pytest

from tests.util import pkg
from oracle import restatement as rs

eng = pkg.engine
pytestmark = pytest.mark.gpu


def _ref(A, W, bias, epi, resid=None):
    ref = A.astype(np.float64) @ W.astype(np.float64).T + bias
    if epi == eng.EPI_BIAS_RESID_F32:
        ref = ref + resid
    ref = ref.astype(np.float32)
    if epi == eng.EPI_BIAS_F16:
        ref = ref.astype(np.float16).astype(np.float32)
    if epi == eng.EPI_BIAS_GELU_F16:
        ref = rs.gelu_table(ref)  # f16(gelu(f32(f16(x)))) -- ggml.c:1434-1441 table semantics
    return ref


# shapes: single tile; M/N/K tails (TMA zero fill + predicated stores); ViT-tiny/base layer shapes; head N=1000
CASES = [
    (128, 256, 64, eng.EPI_BIAS_F32), (128, 128, 64, eng.EPI_BIAS_F32), (128, 256, 64, eng.EPI_BIAS_F16), (1, 128, 64, eng.EPI_BIAS_F32),
    (129, 384, 192, eng.EPI_BIAS_F32), (300, 576, 192, eng.EPI_BIAS_F16), (300, 576, 192, eng.EPI_BIAS_GELU_F16),
    (300, 576, 192, eng.EPI_BIAS_RESID_F32), (197 * 3, 768, 768, eng.EPI_BIAS_RESID_F32), (197 * 3, 3072, 768, eng.EPI_BIAS_GELU_F16),
    (197 * 2, 768, 3072, eng.EPI_BIAS_RESID_F32), (197 * 2, 2304, 768, eng.EPI_BIAS_F16), (256, 1000, 768, eng.EPI_BIAS_F32),
    (7, 1000, 192, eng.EPI_BIAS_F32), (640, 128, 640, eng.EPI_BIAS_RESID_F32),
    (129, 384, 8, eng.EPI_BIAS_F32), (300, 576, 72, eng.EPI_BIAS_F16), (300, 576, 80, eng.EPI_BIAS_GELU_F16),
    (197 * 2, 1152, 4304, eng.EPI_BIAS_RESID_F32),
]


@pytest.mark.parametrize("M,N,K,epi", CASES)
def test_gemm_against_numpy(M, N, K, epi):
    rng = np.random.default_rng(M * 7 + N * 3 + K + epi)
    A = rng.standard_normal((M, K)).astype(np.float16)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((M, N)).astype(np.float32) if epi == eng.EPI_BIAS_RESID_F32 else None
    out = eng.test_gemm(M, N, K, epi, A, W, bias, resid)
    ref = _ref(A, W, bias, epi, resid)
    pre = (A.astype(np.float64) @ W.astype(np.float64).T + bias).astype(np.float32)
    if epi in (eng.EPI_BIAS_RESID_F32, eng.EPI_BIAS_F32):  # f32 outputs: only fp32 accumulation-order noise
        np.testing.assert_allclose(out, ref, rtol=0, atol=2e-5 * max(1.0, np.abs(ref).max()))
    else:  # f16 outputs: identical except where fp32 noise flips an f16 rounding (<= 1 ulp, rare)
        # bias epilogue: at most one f16 ulp.  GELU: a flipped rounding of the f16 INPUT moves the output by up to
        # |slope| (<= 1.13) input ulps, plus half an output ulp for the final rounding -> 2.5 * 2^-10 * max(|x|, |y|)
        ulp = np.maximum(np.maximum(np.abs(ref), np.abs(pre) * (2.5 if epi == eng.EPI_BIAS_GELU_F16 else 0.0)), 2.0 ** -14) * 2.0 ** -10
        noise = 2e-5 * max(1.0, np.abs(ref).max())  # fp32 accumulation noise dominates near zero
        assert (np.abs(out - ref) <= ulp * 1.001 + noise).all()
        assert (out != ref).mean() < 0.02


@pytest.mark.parametrize("M,N,K", [(300, 576, 192), (197 * 3, 2304, 768), (129, 384, 192)])
def test_gemm_split_precision_epilogue(M, N, K):
    """EPI_BIAS_F16_HILO (the qkv GEMM in front of the split-precision attention): hi = f16(x), lo = f16(x - hi); hi + lo must carry the
    f32 result to ~2^-21 relative (2^-24 absolute once lo is subnormal), i.e. only fp32 accumulation-order noise remains."""
    rng = np.random.default_rng(M + N + K)
    A = rng.standard_normal((M, K)).astype(np.float16)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = rng.standard_normal(N).astype(np.float32)
    out = eng.test_gemm(M, N, K, eng.EPI_BIAS_F16_HILO, A, W, bias)
    ref = (A.astype(np.float64) @ W.astype(np.float64).T + bias).astype(np.float32)
    hi, lo = eng.split_hi_lo(ref)
    want = hi.astype(np.float32) + lo.astype(np.float32)
    assert np.abs(want - ref).max() <= 2.0 ** -21 * np.abs(ref).max()      # the representation itself
    np.testing.assert_allclose(out, ref, rtol=0, atol=2e-5 * max(1.0, np.abs(ref).max()) * 0.1 + 2.0 ** -20 * np.abs(ref).max())
    # and the hi part alone is exactly what the plain f16 epilogue writes
    plain = eng.test_gemm(M, N, K, eng.EPI_BIAS_F16, A, W, bias)
    assert (np.abs(out - plain) <= 2.0 ** -11 * np.abs(plain) + 2.0 ** -24).all()


def test_gemm_linearity_at_full_size():
    """Size-independent property at the BASELINE batch size (M = 256*197 = 50432): GEMM(A, W1 + W2) with zero bias equals
    GEMM(A, W1) + GEMM(A, W2) up to fp32 rounding, for exactly representable small-integer operands it is EXACT."""
    M, N, K = 256 * 197, 768, 768
    rng = np.random.default_rng(1)
    A = rng.integers(-4, 5, size=(M, K)).astype(np.float16)
    W1 = rng.integers(-3, 4, size=(N, K)).astype(np.float16)
    W2 = rng.integers(-3, 4, size=(N, K)).astype(np.float16)
    z = np.zeros(N, np.float32)
    o1 = eng.test_gemm(M, N, K, eng.EPI_BIAS_F32, A, W1, z)
    o2 = eng.test_gemm(M, N, K, eng.EPI_BIAS_F32, A, W2, z)
    o12 = eng.test_gemm(M, N, K, eng.EPI_BIAS_F32, A, (W1 + W2), z)
    assert np.array_equal(o1 + o2, o12)  # all partial sums are small integers: exact in fp32
    # spot-check rows from the first, a middle and the last M tile against int64 arithmetic
    for r in (0, 127, 128, 25000, M - 1):
        assert np.array_equal(o1[r].astype(np.int64), A[r].astype(np.int64) @ W1.astype(np.int64).T)



def _scale(hd):
    """The kernels' score scale, the host's 1.0f / sqrtf(hd) in f32: exactly 0.125 at head dim 64."""
    return np.float32(1) / np.sqrt(np.float32(hd))


def _attention_ref(x, B, N, H, hd=64, causal=False):
    """float64 restatement of vit.cpp:826-866 on the values the kernel sees, x [B*N][3*H*hd] (row-major q | k | v: f16 values, or
    hi + lo), with the reference soft-max semantics (ggml.c:10533-10558): s in f32 times the f32 scale, keys past the row at -inf when
    causal (CLIP's text mask), e = f16(exp(f16(s - max))), O = e V / sum e."""
    x = np.asarray(x, np.float64).reshape(B, N, 3, H, hd)
    q, k, v = (x[:, :, i].transpose(0, 2, 1, 3) for i in range(3))
    s = np.einsum("bhqd,bhkd->bhqk", q, k).astype(np.float32) * _scale(hd)
    if causal:
        s = np.where(np.tril(np.ones((N, N), bool)), s, np.float32(-np.inf))
    z = (s - s.max(-1, keepdims=True)).astype(np.float16).astype(np.float64)
    e = np.exp(z).astype(np.float16).astype(np.float64)
    o = np.einsum("bhqk,bhkd->bhqd", e, v) / e.sum(-1, keepdims=True)
    return o.transpose(0, 2, 1, 3).reshape(B * N, H * hd)


@pytest.mark.parametrize("B,N,H", [(3, 17, 2), (2, 197, 3), (1, 224, 1), (40, 197, 12), (2, 50, 1)])
def test_attention_split_precision_against_f32_operand_reference(B, N, H):
    """The wgmma attention kernel with hi + lo operands must follow the f32-operand restatement, not the f16-operand one: a score error of
    2^-12 relative (what rounding q or k to f16 costs) moves x - max across f16 rounding boundaries; with split operands the only
    differences left are f32 accumulation order + the f16 roundings the reference makes too.  The cases cover one to four 64-query
    tiles per problem and many (image, head) problems per launch."""
    rng = np.random.default_rng(N * 7 + H)
    qkv = rng.normal(0.0, 1.0, (B * N, 3 * H * 64)).astype(np.float32)
    qkv[:, : H * 64] *= 1.5
    hi, lo = eng.split_hi_lo(qkv)
    q22 = hi.astype(np.float32) + lo.astype(np.float32)   # the 22-bit values the kernel actually sees
    out = eng.test_attention_hilo(qkv, B, N, H)
    ref = _attention_ref(q22, B, N, H)
    ref16 = _attention_ref(hi, B, N, H)
    assert np.isfinite(out).all()
    err = np.abs(out - ref)
    tol = 2.0 ** -10 * np.abs(ref) + 2e-3 * np.abs(ref).max()
    assert (err <= tol).all(), (err.max(), np.abs(ref).max(), np.unravel_index(err.argmax(), err.shape))
    # closer to the f32-operand result than to the f16-operand one (mean absolute deviation over all outputs)
    assert np.abs(out - ref).mean() < 0.6 * np.abs(out - ref16).mean(), (np.abs(out - ref).mean(), np.abs(out - ref16).mean())


ATTN_CASES = [  # (B, N, H, kernel)
    (3, 17, 2, eng.ATTN_WGMMA), (2, 197, 3, eng.ATTN_WGMMA), (2, 197, 3, eng.ATTN_MMA8),
    (2, 577, 2, eng.ATTN_MMA16), (2, 577, 2, eng.ATTN_MMA8), (1, 225, 1, eng.ATTN_MMA16), (3, 384, 1, eng.ATTN_MMA16),
    (2, 401, 2, eng.ATTN_MMA16), (1, 640, 1, eng.ATTN_MMA16), (20, 577, 16, eng.ATTN_MMA16),
    # 8 warps past the 16-warp kernel's 640 keys, as the engine picks it (ViT-S/8, ViT-B/8: 785 tokens); 896 is the largest token count
    # whose K and V fit in shared memory, the largest request of any attention launch
    (2, 785, 2, eng.ATTN_MMA8), (3, 700, 4, eng.ATTN_AUTO), (1, 896, 1, eng.ATTN_MMA8),
]


@pytest.mark.parametrize("B,N,H,kernel", ATTN_CASES)
def test_attention_kernels_against_numpy(B, N, H, kernel):
    """Every attention kernel, alone, on random QKV (scores spread over several units so the soft-max is not flat): agreement with
    the float64 restatement to f16 output rounding + f32 accumulation noise; the (20, 577, 16) case launches many (image, head)
    problems.  At 896 tokens, one more token is refused by the launcher before anything runs."""
    rng = np.random.default_rng(N * 131 + H)
    qkv = rng.normal(0.0, 1.0, (B * N, 3 * H * 64)).astype(np.float32)
    qkv[:, : H * 64] *= 1.5                       # Q: |s/8| up to ~5
    qkv16 = qkv.astype(np.float16)
    out = eng.test_attention(qkv16, B, N, H, kernel)
    ref = _attention_ref(qkv16, B, N, H)
    assert np.isfinite(out).all()
    err = np.abs(out - ref)
    tol = 2.0 ** -10 * np.abs(ref) + 2e-3 * np.abs(ref).max()
    assert (err <= tol).all(), (err.max(), np.abs(ref).max(), np.unravel_index(err.argmax(), err.shape))
    if N == 896:
        more = rng.normal(0.0, 1.0, (B * 897, 3 * H * 64)).astype(np.float16)
        with pytest.raises(eng.VitB200Error) as ei:
            eng.test_attention(more, B, 897, H, kernel)
        assert "897 tokens do not fit" in str(ei.value) and "max 896" in str(ei.value)


# ---- q8_0 linear layer on the integer tensor cores (prototype, BASELINE.json configs[4]) ---------------------------------------
Q8_CASES = [(128, 128, 128), (1, 128, 128), (300, 576, 768), (197 * 3, 2304, 768), (197 * 2, 768, 3072), (129, 1000, 768), (640, 132, 256)]


@pytest.mark.parametrize("M,N,K", Q8_CASES)
def test_q8_0_gemm_matches_the_reference_integer_dot(M, N, K):
    """wgmma s8 GEMM + on-device activation quantisation against the oracle's quantize_row_q8_0 + vec_dot_q8_0_q8_0
    (bit-exact restatements of the reference, tests/test_oracle.py): the quantised activations (integer work) must be bit-identical,
    the f32 outputs within 1e-5 of the row's largest output (same products, same f32 accumulation, different order of the
    reference's eight partial lanes)."""
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    x = (rng.standard_normal((M, K)) * rng.uniform(0.2, 3.0, (M, 1))).astype(np.float32)
    x[0, :32] = 0.0                                  # an all-zero block: d = 0, id = 0 (ggml-quants.c:733)
    if M > 2:
        x[2, 5] = 1e4                                # an outlier squeezing the rest of its block to a few levels
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    wb = pkg.convert.quantize_q8_0_reference(w.reshape(-1))  # the file quantiser (roundf variant), as `quantize` writes it
    bias = rng.standard_normal(N).astype(np.float32)
    y_ref, xq_ref, xd_ref = rs.linear_q8_0(x, wb, bias)
    y, xq, xd, _ = eng.test_gemm_q8(x, wb, bias)
    assert np.array_equal(xq, xq_ref), "quantised activations differ from quantize_row_q8_0"
    assert np.array_equal(xd.view(np.uint32), xd_ref.view(np.uint32)), "block scales differ from quantize_row_q8_0"
    scale = np.abs(y_ref).max(axis=1, keepdims=True)
    err = (np.abs(y - y_ref) / scale).max()
    assert err <= 1e-5, f"q8_0 GEMM error {err:.3e}"


# ---- LayerNorm: the persistent bulk-copy kernel (D % 128 == 0, >= 8 rows) and the row-per-warp kernel behind the same launcher -----------
@pytest.mark.parametrize("rows,D", [(1, 768), (7, 768), (8, 768), (9, 768), (591, 768), (1154, 1024), (4097, 128), (34, 128), (50, 192), (2, 384),
                                    (591, 256), (591, 384), (57, 512), (4097, 640), (300, 896), (9, 1536), (33, 2048)])
def test_layernorm_matches_the_restatement(rows, D):
    """Row counts around the 8-row block size (partial last block, fewer rows than one block -> row-per-warp kernel), more blocks than
    resident CTAs; hidden sizes of every bulk-copy instantiation (D / 128 = 1 ... 7 float4 per lane) and of every row-per-warp one up to
    the largest accepted hidden size (16 float4 per lane at D = 2048); against the oracle's ggml_norm * w + b rounded to f16 (the GEMM's src1
    conversion): at most one f16 ulp apart (the reference sums in double, the kernel in f32), bit-equal on > 99.5 % of the elements."""
    rng = np.random.default_rng(rows * 131 + D)
    x = (rng.standard_normal((rows, D)) * rng.uniform(0.5, 4.0, (rows, 1)) + rng.uniform(-1, 1, (rows, 1))).astype(np.float32)
    w = rng.uniform(0.5, 1.5, D).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, D).astype(np.float32)
    y = eng.test_layernorm(x, w, b)
    ref = rs.round_f16(rs.layernorm(x, w, b))
    ulp = np.spacing(np.abs(ref).astype(np.float16)).astype(np.float32)
    assert np.isfinite(y).all()
    # one f16 ulp, or -- where (x - mean) * scale * w and b cancel to a result near zero, whose ulp is tiny -- the f32 rounding of the
    # un-cancelled terms (|terms| < 10 here)
    assert (np.abs(y - ref) <= np.maximum(ulp, 4e-6)).all(), float((np.abs(y - ref) / np.maximum(ulp, 4e-6)).max())
    assert (y == ref).mean() > 0.995


# ---- attention kernels at their edges ------------------------------------------------------------------------------------------------
class EdgeForm(NamedTuple):
    """One way the engine runs attention: head dim, heads per image, CLIP's causal mask (query i attends to keys 0 .. i), hi + lo
    operands (split_hi_lo) instead of f16 values, the hook (qkv32 [B*N][3*H*hd], B, N, H) -> [B*N][H*hd], and its token counts.
    The forms of tests/attention_parts.py hand their hook the f16 halves instead: (hi, lo, B, N, H)."""
    hd: int
    H: int
    causal: bool
    split: bool
    run: Callable
    ns: tuple


# Token counts on both sides of every tile boundary of each form.  The wgmma kernel (wgmma on f16 operands, hilo on hi + lo as the
# engine runs it, causal as text towers run it): 64-query tiles and the 224-key box; causal adds 2 (the first row with a masked key) and
# CLIP's 77.  The head-dim-64 mma.sync kernels: 16-query warp tiles, 32-key chunks and the 16-warp kernel's 640-key limit.  The
# head-dim-80 kernel: 16-query warp tiles, 32-key chunks, sweeps of 128 (8 warps, split form, up to 224 tokens) or 256 query rows
# (16 warps, f16 form, 225 to 640 tokens); its three heads put the head slices of a row at 0, 160 and 320 bytes.
_WGMMA_N = (1, 63, 64, 65, 128, 129, 197, 223, 224)
EDGE_FORMS = {
    "wgmma": EdgeForm(64, 2, False, False, lambda x, B, N, H: eng.test_attention(x.astype(np.float16), B, N, H, eng.ATTN_WGMMA), _WGMMA_N),
    "hilo": EdgeForm(64, 2, False, True, eng.test_attention_hilo, _WGMMA_N),
    "mma16": EdgeForm(64, 2, False, False, lambda x, B, N, H: eng.test_attention(x.astype(np.float16), B, N, H, eng.ATTN_MMA16),
                      (129, 160, 640)),
    "mma8": EdgeForm(64, 2, False, False, lambda x, B, N, H: eng.test_attention(x.astype(np.float16), B, N, H, eng.ATTN_MMA8),
                     (1, 31, 32, 33, 641, 896)),
    "hd80split": EdgeForm(80, 3, False, True, lambda x, B, N, H: eng.test_attention_hd(x, B, N, H, 80, True),
                          (1, 15, 16, 17, 31, 32, 33, 127, 128, 129, 197, 223, 224)),
    "hd80f16": EdgeForm(80, 3, False, False, lambda x, B, N, H: eng.test_attention_hd(x, B, N, H, 80, False),
                        (225, 255, 256, 257, 287, 288, 289, 577, 639, 640)),
    "causal": EdgeForm(64, 2, True, True, eng.test_attention_hilo_causal, (1, 2, 63, 64, 65, 77, 128, 129, 193, 224)),
}
EDGE_CASES = [(form, n) for form, f in EDGE_FORMS.items() for n in f.ns]
EDGE_IDS = [f"{form}-N{n}" for form, n in EDGE_CASES]
CAUSAL_CASES = [(form, n) for form, n in EDGE_CASES if EDGE_FORMS[form].causal]
EDGE_B = 3


def _pack(q, k, v):
    """q, k, v [B][N][H][hd] -> the fused [B*N][3*H*hd] buffer the qkv GEMM leaves behind (q heads, then k heads, then v heads)."""
    B, N, H, hd = q.shape
    return np.stack([q, k, v], axis=2).reshape(B * N, 3 * H * hd)


def _run_attention(f, qkv32, B, N):
    return f.run(qkv32, B, N, f.H)


def _operand(f, x32):
    """The value the kernel sees for an f32 operand: f16(x), or hi + lo for the split-precision forms."""
    if f.split:
        hi, lo = eng.split_hi_lo(x32)
        return hi.astype(np.float64) + lo.astype(np.float64)
    return x32.astype(np.float16).astype(np.float64)


def _scores(f, q, k, masked=False):
    """Scaled scores [B][H][i][j] of the operand values in float64 with the f32 scale; -inf past the row if masked and f is causal."""
    s = np.einsum("bihd,bjhd->bhij", _operand(f, q), _operand(f, k)) * np.float64(_scale(f.hd))
    if masked and f.causal:
        s = np.where(np.tril(np.ones(s.shape[-2:], bool)), s, -np.inf)
    return s


# Each case builder asserts its design (score gaps, score ranges, exact operands) before anything is launched, and returns the packed
# input with what the kernel must produce.
def _routing_case(f, N):
    """Keys are random +-1 rows and q_i = 8 k_pi(i): pi is a random permutation of each (image, head), or under the causal mask a
    random key of 0 .. i.  The chosen scaled score (8 hd / sqrt(hd): 64 at hd 64, 71.6 at hd 80) beats every other key of the row by
    >= 20, and f16(exp(x)) is exactly 0 below -17.33, so every probability row is exactly one-hot: output row i is f16(v_pi(i))."""
    B, H, hd = EDGE_B, f.H, f.hd
    rng = np.random.default_rng(1000 + N)
    k = rng.choice(np.array([-1.0, 1.0], np.float32), size=(B, N, H, hd))
    if f.causal:
        pick = rng.integers(0, np.arange(1, N + 1)[:, None], size=(B, N, H))
    else:
        pick = np.stack([np.stack([rng.permutation(N) for _ in range(H)], 1) for _ in range(B)])  # [B][N][H]
    q = np.take_along_axis(k, pick[..., None], axis=1) * 8.0
    v = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    s = _scores(f, q, k, masked=True)
    chosen = np.take_along_axis(s, pick.transpose(0, 2, 1)[..., None], axis=-1)[..., 0]
    assert (chosen == 8.0 * hd * np.float64(_scale(hd))).all()
    if N > 1:
        runner_up = np.sort(s, axis=-1)[..., -2]
        assert (chosen - runner_up >= 20.0).all(), float((chosen - runner_up).min())
    want = np.take_along_axis(_operand(f, v), pick[..., None], axis=1).astype(np.float16).astype(np.float32)
    return _pack(q, k, v), want


def _diagonal_case(f, N):
    """k_j = 20 (j - 112) e_0 and q_i = 8 e_0, exact in f16 (lo = 0) and in the f32 score: scaled score 20 (j - 112).  Unmasked, every
    row's maximum is key N - 1; under the mask row i's is key i and every other key of the row scores >= 20 lower, so output row i is
    f16(v_i).  A mask one key late gives v_(i+1), a missing mask v_(N-1)."""
    B, H, hd = EDGE_B, f.H, f.hd
    rng = np.random.default_rng(5000 + N)
    q = np.zeros((B, N, H, hd), np.float32)
    k = np.zeros((B, N, H, hd), np.float32)
    q[..., 0] = 8.0
    k[..., 0] = 20.0 * (np.arange(N)[:, None] - 112)
    v = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    assert (_operand(f, q) == q).all() and (_operand(f, k) == k).all()
    dot = np.einsum("bihd,bjhd->bhij", q.astype(np.float64), k.astype(np.float64))
    assert (dot.astype(np.float32) == dot).all()
    assert (_scores(f, q, k).argmax(-1) == N - 1).all()
    s = _scores(f, q, k, masked=True)
    assert (s.argmax(-1) == np.arange(N)).all()
    if N > 1:
        top2 = np.sort(s, axis=-1)[..., -2:]
        assert (top2[..., 1] - top2[..., 0] >= 20.0).all()
    return _pack(q, k, v), _operand(f, v).astype(np.float16).astype(np.float32)


def _uniform_case(f, N):
    """q = 0: every score is 0, every e is 1 and output row i is the mean of the V rows it attends to (all N, or 0 .. i under the
    mask).  Tolerance: one f16 output ulp plus the f32 summation error over those n keys."""
    B, H, hd = EDGE_B, f.H, f.hd
    rng = np.random.default_rng(2000 + N)
    q = np.zeros((B, N, H, hd), np.float32)
    k = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    v = (1.0 + 0.5 * rng.standard_normal((B, N, H, hd))).astype(np.float32)
    vs = _operand(f, v)
    if f.causal:
        n = np.arange(1, N + 1)[:, None, None]
        ref, mean_abs = np.cumsum(vs, axis=1) / n, np.cumsum(np.abs(vs), axis=1) / n
    else:
        n = N
        ref, mean_abs = vs.mean(axis=1, keepdims=True), np.abs(vs).mean(axis=1, keepdims=True)
    tol = np.spacing(np.abs(ref).astype(np.float16)).astype(np.float64) + 2 * (n + 2) * 2.0 ** -24 * mean_abs
    return _pack(q, k, v), ref, tol


def _all_negative_case(f, N):
    """Dimension 0 carries -24 after scaling and the rest lies within +-2: every scaled score in [-26, -22], asserted in float64."""
    B, H, hd = EDGE_B, f.H, f.hd
    rng = np.random.default_rng(3000 + N)
    k = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    q = (0.3 * rng.standard_normal((B, N, H, hd))).astype(np.float32)
    k[..., 0], q[..., 0] = 1.0, -24.0 / _scale(hd)
    v = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    s = _scores(f, q, k)
    assert s.min() >= -26.0 and s.max() <= -22.0, (s.min(), s.max())
    qkv = _pack(q, k, v)
    return qkv, _attention_ref(_operand(f, qkv), B, N, H, hd, f.causal)


@pytest.mark.parametrize("form,N", EDGE_CASES, ids=EDGE_IDS)
def test_attention_routes_every_row_exactly(form, N):
    """One-hot probability rows (_routing_case): output row i must be the chosen V row bit for bit.  Every K and V row of every image,
    head, key chunk and query tile must land where it belongs; every attention hook fills its output with NaN first, so a row the
    kernel never writes fails too."""
    f = EDGE_FORMS[form]
    qkv, want = _routing_case(f, N)
    got = _run_attention(f, qkv, EDGE_B, N).reshape(want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (len(bad), bad[:5].tolist())


@pytest.mark.parametrize("form,N", CAUSAL_CASES, ids=[f"{form}-N{n}" for form, n in CAUSAL_CASES])
def test_causal_attention_takes_the_diagonal_only_under_the_mask(form, N):
    """Scores that rise with the key index (_diagonal_case): under the mask each row's largest score is its own key's, so output row i
    must be v_i bit for bit.  An off-by-one or missing mask routes the row to a later key."""
    f = EDGE_FORMS[form]
    qkv, want = _diagonal_case(f, N)
    got = _run_attention(f, qkv, EDGE_B, N).reshape(want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (len(bad), bad[:5].tolist())


@pytest.mark.parametrize("form,N", EDGE_CASES, ids=EDGE_IDS)
def test_attention_uniform_rows_average_exactly_the_real_keys(form, N):
    """Equal scores (_uniform_case) against float64: a padded or foreign key counted in the sum l scales the output by N / N_padded,
    and a key the causal mask should hide changes the mean; both fail."""
    f = EDGE_FORMS[form]
    qkv, ref, tol = _uniform_case(f, N)
    out = _run_attention(f, qkv, EDGE_B, N).reshape(EDGE_B, N, f.H, f.hd)
    err = np.abs(out - ref)
    assert (err <= tol).all(), float((err / tol).max())


@pytest.mark.parametrize("form,N", EDGE_CASES, ids=EDGE_IDS)
def test_attention_all_negative_scores(form, N):
    """Every real scaled score in [-26, -22] (_all_negative_case): against the float64 restatement at the usual tolerance.  A
    zero-filled padding key (score 0) that escaped the masking would become the row maximum, which makes f16(exp) of every real key 0
    (l = 0, NaN output), or, counted in l, add e = f16(exp(>= 22)) = Inf to it (output 0)."""
    f = EDGE_FORMS[form]
    qkv, ref = _all_negative_case(f, N)
    out = _run_attention(f, qkv, EDGE_B, N)
    err = np.abs(out - ref)
    tol = 2.0 ** -10 * np.abs(ref) + 2e-3 * np.abs(ref).max()
    assert (err <= tol).all(), (err.max(), np.abs(ref).max())


@pytest.mark.parametrize("form,N", EDGE_CASES, ids=EDGE_IDS)
def test_attention_non_finite_values_stay_in_their_image(form, N):
    """NaN, then +Inf, in the Q rows, then the K rows, then the V rows of one image or sequence (first, middle, last of three): every
    other one's output is bit-identical to the same launch with that one clean."""
    f = EDGE_FORMS[form]
    B, H = EDGE_B, f.H
    rng = np.random.default_rng(4000 + N)
    qkv = rng.normal(0.0, 1.0, (B, N, 3, H, f.hd)).astype(np.float32)
    clean = _run_attention(f, qkv.reshape(B * N, -1), B, N).reshape(B, N, -1)
    assert np.isfinite(clean).all()
    for val in (np.nan, np.inf):
        for part in range(3):
            for img in range(B):
                x = qkv.copy()
                x[img, :, part] = val
                out = _run_attention(f, x.reshape(B * N, -1), B, N).reshape(B, N, -1)
                others = [b for b in range(B) if b != img]
                assert np.array_equal(out[others], clean[others]), (val, "qkv"[part], img)


# ---- the classifier's soft-max + top-k kernel -------------------------------------------------------------------------------------------
# Inputs x (exact f16 values) where the kernel's f16(exp(x)) differs from the reference's f16 exp table: ex2.approx may land one f16 ulp
# from expf.  {f16 bits of x: f16 bits of the kernel's exp(x)}, as measured on an H100 (NVIDIA H100 80GB HBM3).  Both inputs have
# exp(x) within 2^-3 f16 ulp of a rounding midpoint: exp(-2.615234375) = 0.0731506..., table 0.07318115, kernel 0.07312012;
# exp(-2.966796875) = 0.0514679..., table 0.05148315, kernel 0.05145264.
EXP_ULP_OFF = {0xC13B: 0x2CAE, 0xC1EF: 0x2A96}


def _kernel_exp(x):
    """f16(exp(f16(x))) as the kernel computes it: the reference's table, except at the inputs of EXP_ULP_OFF."""
    e = rs.exp_table(np.asarray(x, np.float32))
    if EXP_ULP_OFF:
        bits = np.asarray(x, np.float32).astype(np.float16).view(np.uint16)
        for xb, eb in EXP_ULP_OFF.items():
            e[bits == xb] = np.array([eb], np.uint16).view(np.float16)[0]
    return e


def test_softmax_exp_of_every_f16_input():
    """One row [0, x_1 .. x_n], the x every f16 value in [-18, 0) (19.6 k classes).  p_0 = 1/sum e exactly, so round_f16(p_i / p_0)
    recovers the kernel's e_i exactly: each must be within one f16 ulp of the reference's exp table, and off by one ulp only at the
    inputs listed in EXP_ULP_OFF.  The probabilities are e * (1/sum e) within the f32 summation error of a float64 computation."""
    bits = np.arange(0x8001, 0xCC81, dtype=np.uint16)       # -2^-24 .. -18
    xs = bits.view(np.float16).astype(np.float32)
    assert xs.min() == -18.0 and xs.max() < 0
    row = np.concatenate([[0.0], xs]).astype(np.float32)[None]
    probs, _, _ = eng.test_softmax_topk(row, 0)
    p0 = np.float64(probs[0, 0])
    e = (probs[0, 1:].astype(np.float64) / p0).astype(np.float16)
    table = rs.exp_table(xs).astype(np.float16)
    off = np.abs(e.view(np.uint16).astype(np.int32) - table.view(np.uint16).astype(np.int32))
    found = {int(b): int(eb) for b, eb in zip(bits[off != 0], e.view(np.uint16)[off != 0])}
    assert off.max() <= 1, int(off.max())
    assert found == EXP_ULP_OFF, f"EXP_ULP_OFF = {found!r}"
    ef = np.concatenate([[1.0], e.astype(np.float64)])
    ref = ef / ef.sum()
    n = row.shape[1]
    assert (np.abs(probs[0] - ref) <= (n / 256 + 32) * 2.0 ** -23 * ref + 1e-45).all()


def _softmax_ref(x):
    """float64 soft-max with the kernel's f16 exp of the f32 difference x - max."""
    z = (x - x.max(axis=1, keepdims=True)).astype(np.float32)
    e = _kernel_exp(z).astype(np.float64)
    return e / e.sum(axis=1, keepdims=True)


def _topk_ref(probs, k):
    """Top-k of the kernel's own probabilities: descending, lowest index first among equals, (-1, 0) past the class count."""
    rows, C = probs.shape
    idx = np.full((rows, k), -1, np.int32)
    val = np.zeros((rows, k), np.float32)
    order = np.lexsort((np.broadcast_to(np.arange(C), probs.shape), -probs.astype(np.float64)), axis=1)[:, :min(k, C)]
    idx[:, :order.shape[1]] = order
    val[:, :order.shape[1]] = np.take_along_axis(probs, order, axis=1)
    return idx, val


SOFTMAX_CASES = [(3, 1, 0), (3, 1, 1), (2, 1, 16), (5, 2, 2), (5, 2, 3), (7, 255, 5), (7, 256, 16), (300, 257, 5), (4, 1000, 16),
                 (300, 1001, 1), (3, 21843, 5), (2, 60000, 16), (2, 60000, 0)]


@pytest.mark.parametrize("rows,C,k", SOFTMAX_CASES)
def test_softmax_topk_class_counts(rows, C, k):
    """Class counts around the 256-thread stride and the pitch padding (NaN in the padding columns must not be read), ImageNet heads,
    21843 classes in shared memory and 60000 on the global scratch path; k from 0 to 16 with k = C and k > C."""
    rng = np.random.default_rng(rows * 7 + C + k)
    x = (3.0 * rng.standard_normal((rows, C))).astype(np.float32)
    probs, idx, val = eng.test_softmax_topk(x, k)
    ref = _softmax_ref(x)
    assert (np.abs(probs - ref) <= (C / 256 + 32) * 2.0 ** -23 * ref + 1e-45).all()
    want_i, want_v = _topk_ref(probs, k)
    assert np.array_equal(idx, want_i) and np.array_equal(val, want_v)


def test_softmax_topk_ties():
    """Equal maxima at indices held by different threads and warps (and by one thread in two strides): lowest index first.  An all-equal
    row: indices 0 .. k-1, equal probabilities."""
    C, k = 1000, 8
    rng = np.random.default_rng(5)
    x = rng.standard_normal((2, C)).astype(np.float32)
    tied = [999, 300, 259, 37, 3]
    x[0, tied] = 6.0
    x[1] = 0.25
    probs, idx, val = eng.test_softmax_topk(x, k)
    assert idx[0, :5].tolist() == sorted(tied) and (val[0, :5] == val[0, 0]).all() and val[0, 5] < val[0, 0]
    assert idx[1].tolist() == list(range(k)) and (val[1] == probs[1, 0]).all() and (probs[1] == probs[1, 0]).all()
    want_i, want_v = _topk_ref(probs, k)
    assert np.array_equal(idx, want_i) and np.array_equal(val, want_v)


def test_softmax_topk_non_finite_rows():
    """A NaN row, a row with a +Inf logit (Inf - Inf is NaN) and a row with -Inf logits among finite ones, each next to finite rows:
    the finite rows are bit-identical to a launch without the others, the -Inf classes get probability 0, and a NaN row gets k entries
    (-1, 0) -- never an index outside [0, C)."""
    C, k = 1001, 5
    rng = np.random.default_rng(6)
    x = (3.0 * rng.standard_normal((7, C))).astype(np.float32)
    x[1, 17] = np.nan
    x[3, 500] = np.inf
    x[5, [0, 255, 256, 1000]] = -np.inf
    probs, idx, val = eng.test_softmax_topk(x, k)
    finite = [0, 2, 4, 6]
    p_f, i_f, v_f = eng.test_softmax_topk(x[finite], k)
    assert np.array_equal(probs[finite], p_f) and np.array_equal(idx[finite], i_f) and np.array_equal(val[finite], v_f)
    for r in (1, 3):
        assert (idx[r] == -1).all() and (val[r] == 0).all(), (r, idx[r].tolist())
    assert (probs[5, [0, 255, 256, 1000]] == 0).all() and np.isfinite(probs[5]).all() and abs(float(probs[5].sum()) - 1) < 1e-3
    ok = [0, 2, 4, 5, 6]
    want_i, want_v = _topk_ref(probs[ok], k)
    assert np.array_equal(idx[ok], want_i) and np.array_equal(val[ok], want_v)
    assert ((idx == -1) | ((idx >= 0) & (idx < C))).all()
