"""The head-dim-72 attention kernel (SigLIP So400m) at its edges: tests/test_gpu_kernels.py's edge suite -- routing, uniform rows,
all-negative scores and non-finite isolation -- on its split-precision form (up to 224 tokens) and its f16 form (225 to 800), and the
lo halves of the split form where head dim 72 adds code: the k8 step of S = Q K^T (columns 64..71, its Ql Kh and Qh Kl products) and the
ninth n8 tile of O = P V (its P Vl product)."""
import numpy as np
import pytest

from tests.util import pkg
from tests.test_gpu_kernels import (EDGE_B, EdgeForm, _all_negative_case, _attention_ref, _operand, _routing_case, _run_attention,
                                    _scale, _uniform_case)

eng = pkg.engine
pytestmark = pytest.mark.gpu

# 16-query warp tiles, 32-key chunks, sweeps of 128 (8 warps, split form, up to 224 tokens) or 256 query rows (16 warps, f16 form, 225 to
# 800 tokens); three heads put the head slices of a row at 0, 144 and 288 bytes
FORMS = {
    "hd72split": EdgeForm(72, 3, False, True, lambda x, B, N, H: eng.test_attention_hd72(x, B, N, H, True),
                          (1, 15, 16, 17, 31, 32, 33, 127, 128, 129, 197, 223, 224)),
    "hd72f16": EdgeForm(72, 3, False, False, lambda x, B, N, H: eng.test_attention_hd72(x, B, N, H, False),
                        (225, 255, 256, 257, 287, 288, 289, 577, 729, 799, 800)),
}
CASES = [(form, n) for form, f in FORMS.items() for n in f.ns]
IDS = [f"{form}-N{n}" for form, n in CASES]


@pytest.mark.parametrize("form,N", CASES, ids=IDS)
def test_routes_every_row_exactly(form, N):
    f = FORMS[form]
    qkv, want = _routing_case(f, N)
    got = _run_attention(f, qkv, EDGE_B, N).reshape(want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (len(bad), bad[:5].tolist())


@pytest.mark.parametrize("form,N", CASES, ids=IDS)
def test_uniform_rows_average_exactly_the_real_keys(form, N):
    f = FORMS[form]
    qkv, ref, tol = _uniform_case(f, N)
    out = _run_attention(f, qkv, EDGE_B, N).reshape(EDGE_B, N, f.H, f.hd)
    err = np.abs(out - ref)
    assert (err <= tol).all(), float((err / tol).max())


@pytest.mark.parametrize("form,N", CASES, ids=IDS)
def test_all_negative_scores(form, N):
    """Every scaled score in [-26, -22]: the f16 exponentials near the bottom of their range, and a padding key that escaped the
    masking would become the row maximum."""
    f = FORMS[form]
    qkv, ref = _all_negative_case(f, N)
    out = _run_attention(f, qkv, EDGE_B, N)
    err = np.abs(out - ref)
    tol = 2.0 ** -10 * np.abs(ref) + 2e-3 * np.abs(ref).max()
    assert (err <= tol).all(), (err.max(), np.abs(ref).max())


@pytest.mark.parametrize("form,N", CASES, ids=IDS)
def test_non_finite_values_stay_in_their_image(form, N):
    f = FORMS[form]
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


@pytest.mark.parametrize("B,N,H", [(3, 17, 2), (2, 197, 3), (1, 224, 1), (8, 197, 16)])
def test_split_precision_follows_the_f32_operand_reference(B, N, H):
    """As test_gpu_kernels' head-dim-64 check: the split form within the usual tolerance of the float64 restatement on hi + lo, and
    closer to it than to the restatement on the f16 values alone."""
    rng = np.random.default_rng(N * 7 + H)
    qkv = rng.normal(0.0, 1.0, (B * N, 3 * H * 72)).astype(np.float32)
    qkv[:, : H * 72] *= 1.5
    hi, lo = eng.split_hi_lo(qkv)
    out = eng.test_attention_hd72(qkv, B, N, H, True)
    ref = _attention_ref(hi.astype(np.float32) + lo.astype(np.float32), B, N, H, 72)
    ref16 = _attention_ref(hi, B, N, H, 72)
    err = np.abs(out - ref)
    assert (err <= 2.0 ** -10 * np.abs(ref) + 2e-3 * np.abs(ref).max()).all(), err.max()
    assert np.abs(out - ref).mean() < 0.6 * np.abs(out - ref16).mean(), (np.abs(out - ref).mean(), np.abs(out - ref16).mean())


SPLIT = FORMS["hd72split"]
TAIL = 64   # the first column of the k8 step and of the ninth n8 tile


def _pack(q, k, v):
    B, N, H, hd = q.shape
    return np.stack([q, k, v], axis=2).reshape(B * N, 3 * H * hd)


@pytest.mark.parametrize("N", [17, 31])
def test_k8_step_takes_the_lo_halves_of_k(N):
    """Scores from column 64 alone: q = 11008 (exact in f16), k_j = 1024 + lo_j with lo_j distinct multiples of 2^-6 below 0.5, so
    hi(k_j) = 1024 for every key.  Only Qh Kl separates the keys, by >= 20 after scaling: each row is one-hot on the key of the largest
    lo, and its output is that key's v bit for bit.  Without Qh Kl every score ties and the output is the mean of v."""
    B, H, hd = 2, 3, 72
    rng = np.random.default_rng(N)
    q = np.zeros((B, N, H, hd), np.float32)
    k = np.zeros((B, N, H, hd), np.float32)
    q[..., TAIL] = 11008.0
    lo = np.stack([np.stack([rng.permutation(N) for _ in range(H)], 1) for _ in range(B)]) * 2.0 ** -6   # [B][N][H]
    k[..., TAIL] = 1024.0 + lo
    v = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    hi_k, lo_k = eng.split_hi_lo(k)
    assert (hi_k[..., TAIL] == 1024).all() and np.array_equal(lo_k[..., TAIL].astype(np.float32), lo.astype(np.float32))
    assert 11008.0 * 2.0 ** -6 * _scale(hd) >= 20.0
    pick = lo.argmax(axis=1)                                                            # [B][H]
    want = np.take_along_axis(_operand(SPLIT, v), pick[:, None, :, None], axis=1).astype(np.float16).astype(np.float32)
    got = eng.test_attention_hd72(_pack(q, k, v), B, N, H, True).reshape(B, N, H, hd)
    assert np.array_equal(got, np.broadcast_to(want, got.shape))


@pytest.mark.parametrize("N", [16, 33])
def test_k8_step_takes_the_lo_halves_of_q(N):
    """Scores from columns 64 and 65 alone: q_i = (1024 + a_i, 1024 + b_i) with hi 1024 in both, keys alternate (1024, -1024) and
    (-1024, 1024).  The hi products cancel, so the score is +-1024 (a_i - b_i) scale from Ql Kh alone, |a_i - b_i| = 0.25: a gap
    of 60 between the two kinds of key.  Row i averages the v of its winning kind; without Ql Kh it averages every key."""
    B, H, hd = 2, 3, 72
    rng = np.random.default_rng(100 + N)
    c = rng.integers(0, 62, size=(B, N, H)) * 2.0 ** -8                                 # 0 .. 0.24
    flip = rng.random((B, N, H)) < 0.5
    a, b = np.where(flip, c + 0.25, c), np.where(flip, c, c + 0.25)                     # |a - b| = 0.25, both below 0.49
    q = np.zeros((B, N, H, hd), np.float32)
    k = np.zeros((B, N, H, hd), np.float32)
    q[..., TAIL], q[..., TAIL + 1] = 1024.0 + a, 1024.0 + b
    kind = np.arange(N) % 2                                                             # 0: (+, -), 1: (-, +)
    k[:, :, :, TAIL] = np.where(kind == 0, 1024.0, -1024.0)[None, :, None]
    k[:, :, :, TAIL + 1] = -k[:, :, :, TAIL]
    v = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    hi_q, _ = eng.split_hi_lo(q)
    assert (hi_q[..., TAIL:TAIL + 2] == 1024).all()
    assert 2 * 1024 * 0.25 * _scale(hd) >= 20.0
    vs = _operand(SPLIT, v)
    win = np.where(a > b, 0, 1)                                                         # [B][N][H]
    ref = np.zeros((B, N, H, hd))
    for w in (0, 1):
        mean_w = vs[:, kind == w].mean(axis=1)                                          # [B][H][hd]
        ref = np.where((win == w)[..., None], mean_w[:, None], ref)
    got = eng.test_attention_hd72(_pack(q, k, v), B, N, H, True).reshape(B, N, H, hd)
    mean_abs = np.abs(vs).mean(axis=1, keepdims=True)
    tol = np.spacing(np.abs(ref).astype(np.float16)).astype(np.float64) + 2 * (N + 2) * 2.0 ** -24 * mean_abs
    assert (np.abs(got - ref) <= tol).all(), float((np.abs(got - ref) / tol).max())


@pytest.mark.parametrize("N", [16, 32])
def test_ninth_n8_tile_takes_the_lo_halves_of_v(N):
    """q = 0 (uniform rows).  In columns 64..71 even keys hold x (|x| in [1, 2), so lo(x) is up to 2^-11) and odd keys -hi(x) of the
    key before, in the same 16-key step: the hi halves cancel and the mean of the rows is the mean of the lo halves alone, several
    tolerances away from 0 on average.  Without P Vl those columns would come out 0."""
    B, H, hd = 2, 3, 72
    rng = np.random.default_rng(200 + N)
    q = np.zeros((B, N, H, hd), np.float32)
    k = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    v = rng.standard_normal((B, N, H, hd)).astype(np.float32)
    x = (rng.uniform(1.0, 2.0, (B, N // 2, H, 8)) * rng.choice([-1.0, 1.0], (B, N // 2, H, 8))).astype(np.float32)
    v[:, 0::2, :, TAIL:] = x
    v[:, 1::2, :, TAIL:] = -x.astype(np.float16).astype(np.float32)
    vs = _operand(SPLIT, v)
    ref = vs.mean(axis=1, keepdims=True)
    tol = np.spacing(np.abs(ref).astype(np.float16)).astype(np.float64) + 2 * (N + 2) * 2.0 ** -24 * np.abs(vs).mean(axis=1, keepdims=True)
    assert np.abs(ref[..., TAIL:]).mean() > 3 * tol[..., TAIL:].mean()
    got = eng.test_attention_hd72(_pack(q, k, v), B, N, H, True).reshape(B, N, H, hd)
    assert (np.abs(got - ref) <= tol).all(), float((np.abs(got - ref) / tol).max())
