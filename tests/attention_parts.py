"""Case builders for the lo-half products of the split-precision attention, in pure numpy.  The kernels compute
S = Ql Kh^T + Qh Kl^T + Qh Kh^T and O = P Vl + P Vh.  Each case puts its operands where only one of these products can route the rows,
so the output is exactly the chosen key's value row only when that product reads the right columns and keys.  The hi and lo halves are
independent f16 arrays here (engine.test_attention_parts passes them as given), not x and its rounding residue.

tests/test_gpu_attention_parts.py runs the cases on the GPU; tests/test_attention_parts_cases.py checks on the CPU that each design
tells the right product set from one with the tested product missing or misplaced."""
import numpy as np

from tests.test_gpu_kernels import EDGE_B, EdgeForm, _scale
from tests.util import pkg

eng = pkg.engine

B = EDGE_B
GROUP = 8        # columns per group: one 16-byte chunk of a swizzled 128-byte K row, or one half of an mma.sync k16 fragment
Q_MUL = 128.0    # q = 128 x the chosen key's +-1 pattern: chosen score 1024, every other key <= 128 x 6 = 768
SCORE_PRODUCTS = {"QlKh": ("Ql", "Kh"), "QhKl": ("Qh", "Kl"), "QhKh": ("Qh", "Kh")}
VALUE_PRODUCTS = {"PVl": "Vl", "PVh": "Vh"}
PRODUCTS = tuple(SCORE_PRODUCTS) + tuple(VALUE_PRODUCTS)
LO_OPERAND = {"QlKh": "Ql", "QhKl": "Kl", "PVl": "Vl"}   # the lo half each tested product reads; the only product that reads it


def _parts(hd, causal):
    return lambda hi, lo, B, N, H: eng.test_attention_parts(hi, lo, B, N, H, hd, causal)


# The split-precision forms, their hook taking (hi, lo, B, N, H).  Token counts: for the wgmma kernels both warpgroups and all four
# 64-query tiles; for the row-major kernel 16-query warp tiles, 32-key chunks and the 128-row sweep of its 8 warps.
FORMS = {
    "wgmma": EdgeForm(64, 2, False, True, _parts(64, False), (1, 17, 64, 65, 129, 197, 224)),
    "causal": EdgeForm(64, 2, True, True, _parts(64, True), (1, 17, 64, 65, 129, 197, 224)),
    "hd80split": EdgeForm(80, 3, False, True, _parts(80, False), (1, 16, 33, 128, 129, 197, 224)),
    "hd72split": EdgeForm(72, 3, False, True, _parts(72, False), (1, 16, 33, 128, 129, 197, 224)),
}
# The column-group cases run at three token counts per form: a partial tile, one that takes both warpgroups (wgmma) or a second
# sweep of the 8 warps (row-major), and 224
GROUP_NS = {"wgmma": (17, 129, 224), "causal": (17, 129, 224), "hd80split": (33, 129, 224), "hd72split": (33, 129, 224)}
# (form, N, product, first column of the group): 8 groups at head dim 64, 9 at 72, 10 at 80; and (form, N) for P Vl, every N
GROUP_CASES = [(form, n, p, c) for form, f in FORMS.items() for n in GROUP_NS[form] for p in ("QhKl", "QlKh")
               for c in range(0, f.hd, GROUP)]
GROUP_IDS = [f"{form}-N{n}-{p}-c{c}" for form, n, p, c in GROUP_CASES]
PVL_CASES = [(form, n) for form, f in FORMS.items() for n in f.ns]
PVL_IDS = [f"{form}-N{n}" for form, n in PVL_CASES]


def _pick(rng, N, H, causal):
    """The key each row chooses, [B][N][H].  A random permutation per (image, head), so every key is some row's choice.  Under the
    causal mask: in image 0 row i takes key i (every key again), in the others a random key of 0 .. i."""
    if not causal:
        return np.stack([np.stack([rng.permutation(N) for _ in range(H)], 1) for _ in range(B)])
    pick = rng.integers(0, np.arange(1, N + 1)[:, None], size=(B, N, H))
    pick[0] = np.arange(N)[:, None]
    return pick


def _patterns(rng, N, H):
    """N distinct +-1 patterns of GROUP columns per (image, head), out of the 256: [B][N][H][GROUP]."""
    idx = np.stack([np.stack([rng.choice(2 ** GROUP, N, replace=False) for _ in range(H)], 1) for _ in range(B)])
    return np.where((idx[..., None] >> np.arange(GROUP)) & 1, 1.0, -1.0)


def _take(x, pick):
    return np.take_along_axis(x, pick[..., None], axis=1)


def _f16(x):
    return np.asarray(x).astype(np.float16).astype(np.float64)


def _heads(x):
    """[B][N][H][hd] -> [B][H][N][hd]"""
    return x.transpose(0, 2, 1, 3)


def _dots(f, ops, products):
    """The sum of the listed score products, unscaled, [B][H][i][j] in float64."""
    N = ops["Qh"].shape[1]
    s = np.zeros((B, f.H, N, N))
    for p, (a, b) in SCORE_PRODUCTS.items():
        if p in products:
            s += _heads(ops[a]) @ _heads(ops[b]).swapaxes(-1, -2)
    return s


def _mask(f, s):
    """-inf past the row under the causal mask."""
    if not f.causal:
        return s
    return np.where(np.tril(np.ones(s.shape[-2:], bool)), s, s.dtype.type(-np.inf))


def model(f, ops, products=PRODUCTS):
    """The kernels' arithmetic on the listed products in float64: S from the score products, the reference soft-max of
    test_gpu_kernels._attention_ref (f32 scores times the f32 scale, the causal mask, e = f16(exp(f16(s - max)))), O = e V / sum e
    with V the sum of the listed value halves, rounded to f16 as the kernels store it -> [B][N][H][hd] float32."""
    s = _mask(f, _dots(f, ops, products).astype(np.float32) * _scale(f.hd))
    e = _f16(np.exp(_f16(s - s.max(-1, keepdims=True))))
    v = sum((ops[n] for p, n in VALUE_PRODUCTS.items() if p in products), np.zeros_like(ops["Vh"]))
    o = ((e @ _heads(v)) / e.sum(-1, keepdims=True)).transpose(0, 2, 1, 3)
    return o.astype(np.float16).astype(np.float32)


def pack(ops):
    """The operand halves [B][N][H][hd] -> the hi and lo float16 buffers [B*N][3*H*hd] (row-major q | k | v) the hook takes."""
    def fuse(q, k, v):
        n, H, hd = q.shape[1:]
        return np.stack([q, k, v], axis=2).reshape(B * n, 3 * H * hd).astype(np.float16)
    return fuse(ops["Qh"], ops["Kh"], ops["Vh"]), fuse(ops["Ql"], ops["Kl"], ops["Vl"])


def run(f, ops):
    """The kernel of form f on the case's halves -> [B][N][H][hd] float32."""
    hi, lo = pack(ops)
    N = ops["Qh"].shape[1]
    return f.run(hi, lo, B, N, f.H).reshape(B, N, f.H, f.hd)


def _check_one_hot(f, ops, pick, chosen):
    """Every row's chosen key scores `chosen` (scaled) and beats every other key of the row by >= 20; f16(exp(x)) is exactly 0 below
    -17.33, so every probability row is exactly one-hot.  Ql Kl, which no kernel computes, is 0."""
    s = _mask(f, _dots(f, ops, PRODUCTS) * np.float64(_scale(f.hd)))
    assert (np.take_along_axis(s, pick.transpose(0, 2, 1)[..., None], axis=-1)[..., 0] == chosen).all()
    if s.shape[-1] > 1:
        runner_up = np.sort(s, axis=-1)[..., -2]
        assert (chosen - runner_up >= 20.0).all(), float((chosen - runner_up).min())
    assert not (_heads(ops["Ql"]) @ _heads(ops["Kl"]).swapaxes(-1, -2)).any()


def group_case(f, N, product, c):
    """One score product alone on the 8 columns [c, c + 8).  Each (image, head) gives its N keys distinct +-1 patterns there, and row
    i's query is 128 x the pattern of its chosen key: scaled score 1024 / sqrt(hd) for the chosen key, at most 768 / sqrt(hd) for any
    other (distinct +-1 8-vectors have dot products <= 6), a gap >= 28.6.  product 'QhKl': q in hi only, the patterns in lo(k) only;
    'QlKh': q in lo only, the patterns in hi(k) only.  v lies in hi, every other column and half is 0.  Without the product every score
    is 0 and a row is the mean of v; taken from another column group or key it routes the rows elsewhere.
    -> (ops, want): the six halves [B][N][H][hd] in float64, and output row i = v of its chosen key, [B][N][H][hd] float32."""
    assert product in ("QhKl", "QlKh") and c % GROUP == 0 and c + GROUP <= f.hd
    rng = np.random.default_rng([f.hd, int(f.causal), N, c, product == "QlKh"])
    pick = _pick(rng, N, f.H, f.causal)
    zero = np.zeros((B, N, f.H, f.hd))
    key = zero.copy()
    key[..., c:c + GROUP] = _patterns(rng, N, f.H)
    query = Q_MUL * _take(key, pick)
    v = _f16(rng.standard_normal((B, N, f.H, f.hd)))
    if product == "QhKl":
        ops = dict(Qh=query, Ql=zero, Kh=zero, Kl=key, Vh=v, Vl=zero)
    else:
        ops = dict(Qh=zero, Ql=query, Kh=key, Kl=zero, Vh=v, Vl=zero)
    assert (_f16(query) == query).all()
    _check_one_hot(f, ops, pick, Q_MUL * GROUP * np.float64(_scale(f.hd)))
    return ops, _take(v, pick).astype(np.float32)


def pvl_case(f, N):
    """P Vl alone: the routing of test_gpu_kernels._routing_case through Qh Kh (random +-1 keys over every column, q_i = 8 k of its
    chosen key, scaled gap >= 20), with the keys chosen as _pick chooses them; lo(q) = lo(k) = 0, hi(v) = 0 and lo(v) random f16
    values.  Output row i is lo(v) of its chosen key exactly; every key is some row's choice, so a lo V tile dropped or read at another
    key step or n8 column tile changes some row.  -> (ops, want) as group_case."""
    rng = np.random.default_rng([f.hd, int(f.causal), N, 7])
    pick = _pick(rng, N, f.H, f.causal)
    zero = np.zeros((B, N, f.H, f.hd))
    k = rng.choice([-1.0, 1.0], size=(B, N, f.H, f.hd))
    vl = _f16(rng.standard_normal((B, N, f.H, f.hd)))
    ops = dict(Qh=8.0 * _take(k, pick), Ql=zero, Kh=k, Kl=zero, Vh=zero, Vl=vl)
    _check_one_hot(f, ops, pick, 8.0 * f.hd * np.float64(_scale(f.hd)))
    return ops, _take(vl, pick).astype(np.float32)


def misplaced(ops, product, c=None):
    """The operands a kernel sees when the tested product reads its lo operand from the wrong place, {name: ops}: 'group 0' (every
    column group read from columns 0..7; skipped when the case's group is 0) and 'row 0' (every row read from row 0: key 0, or query 0
    for Ql; skipped at one token).  The lo operand feeds no other product, so only the tested one changes."""
    name = LO_OPERAND[product]
    lo = ops[name]
    out = {}
    if c != 0:
        out["group 0"] = np.tile(lo[..., :GROUP], lo.shape[-1] // GROUP)
    if lo.shape[1] > 1:
        out["row 0"] = np.broadcast_to(lo[:, :1], lo.shape)
    return {m: {**ops, name: x} for m, x in out.items()}
