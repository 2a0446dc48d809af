"""The checks of tests/row_reference.py, without a GPU: each accepts a faithful f32 emulation of its kernel and rejects an output with
the mistake it exists to catch planted in it (a wrong epsilon, a wrong row count or row in a mean, the second EOS or maximum instead of
the first, bf16 by truncation, position rows shifted by one, a neighbouring sequence's pooled row)."""
import numpy as np
import pytest

from tests import row_reference as rr

D_LIST = [64, 320, 576, 1088, 2048]


def _rows(D, eps, seed=0):
    return rr.designed_rows(8, D, eps, np.random.default_rng(seed))


def _params(D, seed=1):
    rng = np.random.default_rng(seed)
    return (1 + 0.2 * rng.standard_normal(D)).astype(np.float32), (0.1 * rng.standard_normal(D)).astype(np.float32)


@pytest.mark.parametrize("D", D_LIST)
@pytest.mark.parametrize("eps", [1e-6, 1e-5])
def test_layernorm_checks(D, eps):
    x = _rows(D, eps)
    w, b = _params(D)
    y = rr.layernorm_f32_emulation(x, w, b, eps)
    assert np.array_equal(y[7], b), "a constant dyadic row normalises to b exactly"
    rr.check_layernorm(y, x, w, b, eps, "f32")
    rr.check_layernorm(y.astype(np.float16), x, w, b, eps, "f16")
    rr.check_layernorm(rr.bf16_rne_bits(y), x, w, b, eps, "bf16")
    bad = rr.layernorm_f32_emulation(x, w, b, 10 * eps)
    for kind, out in (("f32", bad), ("f16", bad.astype(np.float16)), ("bf16", rr.bf16_rne_bits(bad))):
        with pytest.raises(AssertionError):
            rr.check_layernorm(out, x, w, b, eps, kind)
    with pytest.raises(AssertionError):  # bf16 by truncation
        rr.check_layernorm(rr.bf16_trunc_bits(y), x, w, b, eps, "bf16")


def test_rounded_rows_check():
    x = _rows(320, 1e-6, seed=3)
    rr.check_rounded_rows(x.copy(), x, "f32")
    rr.check_rounded_rows(x.astype(np.float16), x, "f16")
    rr.check_rounded_rows(rr.bf16_rne_bits(x), x, "bf16")
    with pytest.raises(AssertionError):
        rr.check_rounded_rows(rr.bf16_trunc_bits(x), x, "bf16")


def _pool_input(B, R, G, D, first_patch, seed=5):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, first_patch + G * G, D)).astype(np.float32)
    x[:, 1:first_patch] += 5  # registers far from the patch rows, so that one in the mean shows
    return x


def _pool_bugs(x, first_patch, lnf):
    """The pool with a planted mistake, in f32 ('lnf' maps the rows first: the LayerNorm or nothing): the mean over N_p - 1 rows,
    divided by the token count N_p + R + 1, and with the last register row included."""
    y = lnf(x)
    B, N, D = y.shape
    n = N - first_patch
    head = [y[:, 0]] if first_patch else []
    out = {"N_p - 1 rows": y[:, first_patch:-1].sum(1, dtype=np.float32) / np.float32(n - 1) if n > 1 else None,
           "divided by N_p + R + 1": y[:, first_patch:].sum(1, dtype=np.float32) / np.float32(N) if first_patch else None,
           "a register row in the mean": y[:, first_patch - 1:].sum(1, dtype=np.float32) / np.float32(n) if first_patch > 1 else None}
    return {k: np.concatenate(head + [v], 1).astype(np.float32) for k, v in out.items() if v is not None}


@pytest.mark.parametrize("R,G,D", [(0, 1, 64), (1, 2, 320), (4, 3, 576), (16, 5, 1088), (16, 29, 2048), (-1, 3, 512), (-1, 29, 64)])
@pytest.mark.parametrize("kind", ["f32", "f16", "bf16"])
def test_pool_checks(R, G, D, kind):
    """R = -1: the mean pool (no class token); otherwise the class-plus-patch-mean pool with R registers."""
    first = 0 if R < 0 else 1 + R
    x = _pool_input(2, R, G, D, first)
    w, b = _params(D)
    out = lambda v: v if kind == "f32" else v.astype(np.float16) if kind == "f16" else rr.bf16_rne_bits(v)
    raw = rr.pool_raw_emulation(x, first)
    rr.check_pool_raw(out(raw), x, first, kind)
    norm = rr.pool_raw_emulation(rr.layernorm_f32_emulation(x, w, b, 1e-6), first)
    rr.check_pool_norm(out(norm), x, first, w, b, 1e-6, kind)
    if kind == "bf16":
        with pytest.raises(AssertionError):
            rr.check_pool_raw(rr.bf16_trunc_bits(raw), x, first, kind)
    bugs_raw = _pool_bugs(x, first, lambda v: v)
    bugs_norm = _pool_bugs(x, first, lambda v: rr.layernorm_f32_emulation(v, w, b, 1e-6))
    assert G == 1 or "N_p - 1 rows" in bugs_raw
    for name in bugs_raw:
        with pytest.raises(AssertionError):
            rr.check_pool_raw(out(bugs_raw[name]), x, first, kind, name)
        with pytest.raises(AssertionError):
            rr.check_pool_norm(out(bugs_norm[name]), x, first, w, b, 1e-6, kind, name)


def test_embed_check():
    rng = np.random.default_rng(7)
    P, C, G, D, R = 8, 3, 3, 64, 4
    imgs = rng.integers(-3, 4, (2, G * P, G * P, C)).astype(np.float32)
    wt = rng.integers(-2, 3, (D, C, P, P)).astype(np.float16)
    bias = rng.integers(-4, 5, D).astype(np.float32)
    pos = (rng.integers(-32, 33, (1 + R + G * G, D)) / 4).astype(np.float32)
    prefix = (rng.integers(-32, 33, (1 + R, D)) / 4).astype(np.float32)
    ref = rr.embed_reference(imgs, wt, bias, pos, prefix, P)
    # a direct convolution, pixel by pixel, gives the same rows
    b, p, d = 1, 5, 9
    py, px = divmod(p, G)
    conv = sum(float(wt[d, c, ky, kx]) * imgs[b, py * P + ky, px * P + kx, c] for c in range(C) for ky in range(P) for kx in range(P))
    assert ref[b, 1 + R + p, d] == conv + bias[d] + pos[1 + R + p, d]
    rr.check_exact(ref.astype(np.float32), ref)
    shifted = rr.embed_reference(imgs, wt, bias, np.roll(pos, 1, axis=0), prefix, P)
    with pytest.raises(AssertionError):
        rr.check_exact(shifted.astype(np.float32), ref)


def test_token_embed_check():
    rng = np.random.default_rng(8)
    V, N, D = 50, 33, 64
    tok = rng.standard_normal((V, D)).astype(np.float16)
    pos = rng.standard_normal((N, D)).astype(np.float32)
    ids = rng.integers(0, V, (3, N))
    ids[0, 0], ids[1, -1] = 0, V - 1
    want = tok.astype(np.float32)[ids] + pos
    rr.check_token_embed(want, ids, tok, pos)
    with pytest.raises(AssertionError):
        rr.check_token_embed(tok.astype(np.float32)[ids] + np.roll(pos, 1, axis=0), ids, tok, pos)
    with pytest.raises(AssertionError):  # the sum in float64, rounded once: not the kernel's f32 add of the f16 value
        rr.check_token_embed((tok.astype(np.float64)[ids] + pos.astype(np.float64) + 1e-7).astype(np.float32), ids, tok, pos)


def test_text_pool_rule():
    assert rr.text_pool_row([5, 7, 3, 7], "eos", 7) == 1
    assert rr.text_pool_row([5, 6, 3], "eos", 7) == 0
    assert rr.text_pool_row([5, 9, 3, 9, 9], "eos_argmax", 7) == 1
    assert rr.text_pool_row([5, 9, 3], "last", 7) == 2


@pytest.mark.parametrize("pool", ["eos", "eos_argmax"])
def test_text_pool_check(pool):
    rng = np.random.default_rng(9)
    B, N, D, V, eos = 4, 40, 128, 100, 7
    ids = rng.integers(8, V - 1, (B, N))
    end = eos if pool == "eos" else V - 1
    for s, start in enumerate([3, 30, 31, 33]):
        ids[s, start:] = end  # padded with the end id: every position from `start` on ties
    x = rng.standard_normal((B, N, D)).astype(np.float32)
    w, b = _params(D)
    y = rr.layernorm_f32_emulation(x, w, b, 1e-5)
    rows = [rr.text_pool_row(s, pool, eos) for s in ids]
    pick = lambda r: np.stack([y[s, r[s]] for s in range(B)]).astype(np.float16).astype(np.float32)
    rr.check_text_pool(pick(rows), x, ids, pool, eos, w, b, 1e-5)
    with pytest.raises(AssertionError):  # the second EOS / maximum
        rr.check_text_pool(pick([r + 1 for r in rows]), x, ids, pool, eos, w, b, 1e-5)
    with pytest.raises(AssertionError):  # a neighbouring sequence's pooled row
        good = pick(rows)
        rr.check_text_pool(np.roll(good, 1, axis=0), x, ids, pool, eos, w, b, 1e-5)


def test_logits_bound():
    rng = np.random.default_rng(10)
    a = rng.standard_normal((3, 256)).astype(np.float16)
    W = (0.05 * rng.standard_normal((10, 256))).astype(np.float16)
    bias = rng.standard_normal(10).astype(np.float32)
    ref, bound = rr.logits_bound(a, W, bias)
    f32 = (a.astype(np.float32) @ W.astype(np.float32).T + bias).astype(np.float32)
    rr.check_f32(f32, ref, bound)
    with pytest.raises(AssertionError):  # logits of the wrong row
        rr.check_f32(f32[::-1], ref, bound)
