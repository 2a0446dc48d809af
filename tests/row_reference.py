"""Float64 references, and element-by-element checks against them, for the kernels at the two ends of a forward pass: the embedding
stage (cls_rows_kernel and the patch GEMM's `+ pos`), the row LayerNorm (layernorm_f16_kernel, layernorm_inplace_kernel), the
class-plus-patch-mean and mean pools (cls_patch_mean_kernel), the token gather (token_embed_kernel) and the text pool (text_pool_kernel).
It needs no GPU: tests/test_gpu_row_kernels.py holds the kernels' outputs to these checks, tests/test_row_reference.py shows that each
check rejects the mistake it exists for.

Bounds (u = 2^-24, the f32 unit roundoff), derived from the kernels' operation counts in csrc/kernels.cuh:

LayerNorm (ln_center + ln_affine).  A row sum passes through at most 2 adds in sum4, MAXV <= 16 lane accumulations and 5 butterfly
steps, then one division: |mean - mu| <= delta = 32 u mean|x| (24 operations, rounded up).  The centred values are
(x - mu - delta)(1 + u), so the output moves by at most delta scale |w| through the mean.  The squares' sum has the same 24 levels plus
the square: its relative error is <= 26 u, and since the centred values are off by delta the computed variance is var + delta^2 (the
cross term sums to zero).  `+ eps`, `/ D`, sqrtf and 1 / x add 4 roundings, so scale is off by <= 15 u relative plus
delta^2 scale^2 / 2.  The three rounded ops of the affine add 3 u.  With t = (x - mu) scale w and y = t + b:
    |y - y64| <= 64 u (|t| + |y64|) + delta scale |w| + delta^2 scale^2 |t|
(64 u covers the ~20 u of relative error with room for the f32 rounding of every intermediate; the last term is the variance's, which
matters only where |mean| >> sigma).

Means of LayerNorm rows (cls_patch_mean_kernel, NORM).  Each warp adds ceil(N_p / 8) rows, the 8 partials are added in 7 steps and
divided once: (ceil(N_p / 8) + 9) u mean|y| on top of the mean of the rows' own bounds.

16-bit outputs are the round-to-nearest-even of the f32 value, so a kernel output is correct when it is the 16-bit rounding of some
value within the f32 bound of the float64 result: between the roundings of y64 - bound and y64 + bound.  Where the bound is below half
a 16-bit ulp (nearly everywhere) that is one value or its neighbour, i.e. within one ulp of the rounding of y64.

Where the kernel pins every rounding with __fadd_rn / __fdiv_rn (the un-normalised pool, the embedding sums, the token gather) the
checks demand bit equality with numpy's f32 arithmetic in the kernel's order."""
import numpy as np

U = 2.0 ** -24
POOL_WARPS = 8  # csrc/kernels.cuh POOL_WARPS: one CTA of 8 warps per image


# ------------------------------------------------------------------------------------------------
# 16-bit roundings and their ordering

def bf16_rne_bits(x) -> np.ndarray:
    """f32 -> bf16 bit patterns, round to nearest even (finite values)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_trunc_bits(x) -> np.ndarray:
    """f32 -> bf16 bit patterns by truncation (a wrong rounding, for the checks' self-test)."""
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) >> 16).astype(np.uint16)


def bits16(x, kind: str) -> np.ndarray:
    """f32 values -> their 16-bit RNE bit patterns; kind 'f16' or 'bf16'."""
    x = np.ascontiguousarray(x, np.float32)
    return x.astype(np.float16).view(np.uint16) if kind == "f16" else bf16_rne_bits(x)


def as_bits16(got, kind: str) -> np.ndarray:
    """A kernel's 16-bit output (float16 values, or bf16 as the uint16 bit patterns the features API returns) -> bit patterns."""
    got = np.asarray(got)
    if kind == "f16":
        return np.ascontiguousarray(got, np.float16).view(np.uint16)
    assert got.dtype == np.uint16
    return got


def _ordinal(bits) -> np.ndarray:
    """16-bit patterns -> integers in the order of their values (+0 and -0 both 0): neighbouring values differ by 1."""
    b = np.asarray(bits, np.uint16).astype(np.int64)
    return np.where(b & 0x8000, -(b & 0x7FFF), b)


def _f32_down(v):
    v = np.asarray(v, np.float64)
    f = v.astype(np.float32)
    return np.where(f.astype(np.float64) > v, np.nextafter(f, np.float32(-np.inf)), f)


def _f32_up(v):
    v = np.asarray(v, np.float64)
    f = v.astype(np.float32)
    return np.where(f.astype(np.float64) < v, np.nextafter(f, np.float32(np.inf)), f)


def check_round16(got, ref, bound, kind: str, what: str = ""):
    """got (16-bit) must be the RNE of a value within `bound` of the float64 `ref`: between the roundings of ref - bound and ref + bound
    (each first rounded outward to f32, which keeps the interval a superset)."""
    o = _ordinal(as_bits16(got, kind))
    lo = _ordinal(bits16(_f32_down(np.asarray(ref) - bound), kind))
    hi = _ordinal(bits16(_f32_up(np.asarray(ref) + bound), kind))
    bad = (o < lo) | (o > hi)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} {kind} values outside the rounding of the bound, first at " \
                          f"{np.argwhere(bad)[0].tolist()}"


def check_f32(got, ref, bound, what: str = ""):
    err = np.abs(np.asarray(got, np.float64) - ref)
    bad = ~(err <= bound)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} values outside the bound, worst err / bound " \
                          f"{float(np.max(err / np.maximum(bound, 1e-300))):.3g}"


def check_output(got, ref, bound, kind: str, what: str = ""):
    """An f32 ('f32') or 16-bit output against ref +- bound."""
    if kind == "f32":
        check_f32(got, ref, bound, what)
    else:
        check_round16(got, ref, bound, kind, what)


def check_rounded_rows(got, x, kind: str, what: str = ""):
    """An un-normalised output: exactly the observed f32 rows x, or their RNE to 16 bits."""
    x = np.ascontiguousarray(x, np.float32)
    if kind == "f32":
        ok = np.array_equal(np.asarray(got, np.float32).view(np.uint32), x.view(np.uint32))
    else:
        ok = np.array_equal(as_bits16(got, kind), bits16(x, kind))
    assert ok, f"{what}: not the {kind} rounding of the rows, bit for bit"


# ------------------------------------------------------------------------------------------------
# LayerNorm

def layernorm_bound(x, w, b, eps):
    """(y64, bound): the float64 LayerNorm of the f32 rows x [..., D] with the f32 parameters, and the f32 kernel's error bound (module
    docstring).  eps is taken as the f32 value the engine holds."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float32).astype(np.float64).reshape(-1)
    b = np.asarray(b, np.float32).astype(np.float64).reshape(-1)
    e = float(np.float32(eps))
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    scale = 1.0 / np.sqrt(var + e)
    t = (x - mu) * scale * w
    y = t + b
    delta = 32 * U * np.abs(x).mean(-1, keepdims=True)
    bound = 64 * U * (np.abs(t) + np.abs(y)) + delta * scale * np.abs(w) + delta ** 2 * scale ** 2 * np.abs(t)
    return y, bound


def _maxv(D: int) -> int:
    return 4 if D <= 512 else 8 if D <= 1024 else 16


def _warp_sum(p):
    """The kernel's butterfly over the last axis (32 lanes), in f32: every lane ends with the same sum; lane 0's is returned."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        p = p + p[..., lanes ^ o]
    return p[..., 0]


def layernorm_f32_emulation(x, w, b, eps):
    """The row LayerNorm in numpy f32 in the kernel's order (ln_center, ln_affine): float4 l + 32 j of a row in lane l, per-lane sums
    of ((x + y) + (z + w)), the butterfly, f32 division, sqrtf and the three rounded affine ops.  Products are not contracted into FMAs
    (nvcc may contract them; that is within the bound either way)."""
    x = np.ascontiguousarray(x, np.float32)
    lead, D = x.shape[:-1], x.shape[-1]
    rows = x.reshape(-1, D)
    nvec, mv = D // 4, _maxv(D)
    v = np.zeros((rows.shape[0], mv * 32, 4), np.float32)
    v[:, :nvec] = rows.reshape(-1, nvec, 4)
    v = v.reshape(-1, mv, 32, 4)  # [row][j][lane][4]: float4 lane + 32 j
    live = (np.arange(32)[None, :] + 32 * np.arange(mv)[:, None] < nvec)[None, :, :, None]
    s = np.zeros(v.shape[:1] + (32,), np.float32)
    for j in range(mv):
        s = s + ((v[:, j, :, 0] + v[:, j, :, 1]) + (v[:, j, :, 2] + v[:, j, :, 3]))
    mean = _warp_sum(s) / np.float32(D)
    c = np.where(live, v - mean[:, None, None, None], np.float32(0))
    sq = np.zeros_like(s)
    for j in range(mv):
        q = c[:, j] * c[:, j]
        sq = sq + ((q[..., 0] + q[..., 1]) + (q[..., 2] + q[..., 3]))
    scale = np.float32(1) / np.sqrt(_warp_sum(sq) / np.float32(D) + np.float32(eps))
    c = c.reshape(-1, mv * 32 * 4)[:, :D]
    y = (c * scale[:, None]) * np.asarray(w, np.float32).reshape(-1) + np.asarray(b, np.float32).reshape(-1)
    return y.reshape(lead + (D,)).astype(np.float32)


def check_layernorm(got, x, w, b, eps, kind: str, what: str = ""):
    """A normalised output (f32, f16 or bf16) of the f32 rows x."""
    y, bound = layernorm_bound(x, w, b, eps)
    check_output(got, y, bound, kind, what)


def designed_rows(n: int, D: int, eps: float, rng) -> np.ndarray:
    """n f32 rows of D whose statistics are the LayerNorm's edges, row r of kind r % 8: variance 2 eps and 8 eps (where eps matters),
    |mean| / sigma = 1e3 and 1e2, sigma 1e-3, 1e2 and 1, and a row constant at the dyadic 0.75 (its sum is exact: it normalises to b)."""
    z = rng.standard_normal((n, D))
    z = (z - z.mean(1, keepdims=True)) / z.std(1, keepdims=True)
    sig = np.array([np.sqrt(2 * eps), np.sqrt(8 * eps), 0.1, 1e-3, 1e2, 1.0, 0.3, 0.0])[np.arange(n) % 8, None]
    mean = np.array([0.0, 0.0, 100.0, 0.0, 0.0, 0.5, -30.0, 0.75])[np.arange(n) % 8, None]
    return (mean + sig * z).astype(np.float32)


# ------------------------------------------------------------------------------------------------
# The class-plus-patch-mean and mean pools (cls_patch_mean_kernel)

def pool_raw_emulation(x, first_patch: int) -> np.ndarray:
    """NORM = false, f32, in the kernel's order: x [B][N][D] f32 -> [B][D] (first_patch = 0) or [B][2 D] (row 0 || the mean).  Warp w
    adds rows first_patch + w, + 8, ... from 0.0f; the eight partials are added warp 0 first, then divided by the patch count."""
    x = np.ascontiguousarray(x, np.float32)
    B, N, D = x.shape
    parts = np.zeros((POOL_WARPS, B, D), np.float32)
    for w in range(POOL_WARPS):
        for r in range(first_patch + w, N, POOL_WARPS):
            parts[w] = parts[w] + x[:, r]
    s = parts[0]
    for k in range(1, POOL_WARPS):
        s = s + parts[k]
    mean = s / np.float32(N - first_patch)
    return np.concatenate([x[:, 0], mean], axis=1) if first_patch > 0 else mean


def check_pool_raw(got, x, first_patch: int, kind: str, what: str = ""):
    """The un-normalised pool: bit for bit the f32 emulation, rounded to the output type."""
    check_rounded_rows(got, pool_raw_emulation(x, first_patch), kind, what)


def pool_norm_bound(x, first_patch: int, w, b, eps):
    """(ref, bound) of the normalised pool: [LN(row 0) ||] the float64 mean of the float64 LayerNorms of the patch rows."""
    y, bound = layernorm_bound(x, w, b, eps)
    p, pb = y[:, first_patch:], bound[:, first_patch:]
    n = p.shape[1]
    ref = p.mean(1)
    bnd = pb.mean(1) + (-(-n // POOL_WARPS) + 9) * U * (np.abs(p) + pb).mean(1)
    if first_patch > 0:
        ref, bnd = np.concatenate([y[:, 0], ref], 1), np.concatenate([bound[:, 0], bnd], 1)
    return ref, bnd


def check_pool_norm(got, x, first_patch: int, w, b, eps, kind: str, what: str = ""):
    ref, bound = pool_norm_bound(x, first_patch, w, b, eps)
    check_output(got, ref, bound, kind, what)


# ------------------------------------------------------------------------------------------------
# The embedding stage of image towers and of text towers

def patch_rows(imgs, P: int) -> np.ndarray:
    """images [B][S][S][C] (HWC) -> patch rows [B][G*G][C*P*P], k = c P^2 + ky P + kx, patches row-major."""
    imgs = np.asarray(imgs, np.float64)
    if imgs.ndim == 3:
        imgs = imgs[..., None]
    B, S, _, C = imgs.shape
    G = S // P
    return imgs.reshape(B, G, P, G, P, C).transpose(0, 1, 3, 5, 2, 4).reshape(B, G * G, C * P * P)


def embed_reference(imgs, weight, bias, pos, prefix, P: int) -> np.ndarray:
    """Layer-0 token rows in float64: [prefix[r] + pos[r] for r < R] then the conv of each patch + bias + pos[R + p].  weight
    [D][C][P][P], pos [N][D], prefix [R][D] (class token then registers; R = 0 without a class token)."""
    a = patch_rows(imgs, P)
    wt = np.asarray(weight, np.float64).reshape(weight.shape[0], -1)
    pos = np.asarray(pos, np.float64).reshape(-1, wt.shape[0])
    prefix = np.asarray(prefix, np.float64).reshape(-1, wt.shape[0])
    R = prefix.shape[0]
    patches = a @ wt.T + np.asarray(bias, np.float64).reshape(-1) + pos[R:]
    head = np.broadcast_to(prefix + pos[:R], (a.shape[0], R, wt.shape[0]))
    return np.concatenate([head, patches], axis=1)


def check_exact(got, ref, what: str = ""):
    """got (f32) equals ref bit for bit; ref must itself be f32-exact, or the comparison would depend on a rounding."""
    ref = np.asarray(ref, np.float64)
    assert np.array_equal(ref.astype(np.float32).astype(np.float64), ref), f"{what}: the reference is not exact in f32"
    bad = np.asarray(got, np.float32).astype(np.float64) != ref
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} values differ, first at {np.argwhere(bad)[0].tolist()}"


def token_embed_reference(ids, tok16, pos) -> np.ndarray:
    """token_embed_kernel in numpy f32: f32(tok[id]) + pos[t], one rounded add per element."""
    ids = np.asarray(ids)
    t = np.asarray(tok16, np.float16).astype(np.float32)
    p = np.asarray(pos, np.float32).reshape(-1, t.shape[1])
    return t[ids] + p[None, : ids.shape[1]]


def check_token_embed(got, ids, tok16, pos, what: str = ""):
    want = token_embed_reference(ids, tok16, pos)
    got = np.ascontiguousarray(got, np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} values differ, first at {np.argwhere(bad)[0].tolist()}"


# ------------------------------------------------------------------------------------------------
# The text pool

def text_pool_row(seq, pool: str, eos: int) -> int:
    """The pooled position of one sequence: 'eos' the first EOS (0 without one), 'eos_argmax' the first position of the largest id,
    'last' the last position."""
    seq = [int(v) for v in seq]
    if pool == "last":
        return len(seq) - 1
    if pool == "eos":
        return seq.index(eos) if eos in seq else 0
    return seq.index(max(seq))


def check_text_pool(embeds, x, ids, pool: str, eos: int, w, b, eps, what: str = ""):
    """embeds [B][D] (an identity head's output: the f16 pooled rows widened) against the float64 LayerNorm of each sequence's pooled
    row of x [B][N][D].  Every other candidate -- each other row of the sequence, and the pooled row of every other sequence -- must be
    rejected by the same check unless its row is bit-identical, so a wrong row cannot pass."""
    x = np.ascontiguousarray(x, np.float32)
    e16 = np.asarray(embeds, np.float32).astype(np.float16)
    assert np.array_equal(e16.astype(np.float32), np.asarray(embeds, np.float32)), f"{what}: embeds are not f16 values"
    rows = [text_pool_row(s, pool, eos) for s in ids]
    y, bound = layernorm_bound(x, w, b, eps)
    for s, r in enumerate(rows):
        check_round16(e16[s], y[s, r], bound[s, r], "f16", f"{what} sequence {s} row {r}")
        others = [(s, t) for t in range(x.shape[1]) if t != r] + [(q, rows[q]) for q in range(len(rows)) if q != s]
        for q, t in others:
            if np.array_equal(x[q, t].view(np.uint32), x[s, r].view(np.uint32)):
                continue
            o = _ordinal(e16[s].view(np.uint16))
            lo = _ordinal(bits16(_f32_down(y[q, t] - bound[q, t]), "f16"))
            hi = _ordinal(bits16(_f32_up(y[q, t] + bound[q, t]), "f16"))
            assert ((o < lo) | (o > hi)).any(), f"{what}: sequence {s}'s row {r} cannot be told from sequence {q}'s row {t}"


# ------------------------------------------------------------------------------------------------
# The head

def logits_bound(a, W, bias):
    """(ref, bound) of the head GEMM on its f16 A operand: float64 a @ W^T + b with W as the engine holds it (rounded to f16), and the
    f32 accumulation bound of tests/test_gpu_kernels.py::test_gemm_against_numpy (2e-5 of max(1, max |ref|))."""
    W16 = np.asarray(W, np.float32).astype(np.float16)
    ref = np.asarray(a, np.float64) @ W16.astype(np.float64).T + np.asarray(bias, np.float32).astype(np.float64).reshape(-1)
    return ref, 2e-5 * max(1.0, float(np.abs(ref).max()))
