"""The kernels at the two ends of a forward pass, element by element against float64 (tests/row_reference.py): the embedding stage
(cls_rows_kernel, the patch GEMM's `+ pos`), the final LayerNorm of the features (layernorm_f16_kernel with f32 / f16 / bf16 outputs,
normalised or not), the class-plus-patch-mean and mean pools (cls_patch_mean_kernel), the head's A operand and logits, CLIP's pre-norm
(layernorm_inplace_kernel), the token gather (token_embed_kernel) and the text pool (text_pool_kernel).

No extra entry point is needed: each kernel's exact input is observable.  The un-normalised f32 features at depth k are a copy of the
residual stream X that the final LayerNorm and the pools read at that depth; the `x_final` and `final_ln` debug taps are the head's input
and output; a text tower's un-normalised tokens after its last block are what the text pool reads, and with an identity head its embeds
are the pool's f16 output widened; a twin of a CLIP tower without its pre-norm gives the pre-norm's input.  Models have one block and
are built in memory, so the shapes are free within the loader's rules: hidden sizes 64 .. 2048 (every MAXV, half-live and partly live
lanes), 1 .. 841 patches, 0 .. 16 registers, contexts 1 .. 224."""
import functools
import itertools

import numpy as np
import pytest

from tests.util import pkg, gf
from tests import row_reference as rr

eng = pkg.engine
pytestmark = pytest.mark.gpu

D_LIST = [64, 320, 512, 576, 1024, 1088, 2048]
DTYPES = {"f32": np.float32, "f16": np.float16, "bf16": eng.BFLOAT16}
AMPS = [0.0, 1.0, 30.0, 1e-2, 3.0]  # image b's pixels: amplitude AMPS[b] times N(0, 1); image 0 is all zero, its rows are pos_embed's


@functools.lru_cache(maxsize=None)
def _block(D: int) -> dict:
    """One block's weights for hidden size D (shared by every model of that width)."""
    rng = np.random.default_rng(D)
    mat = lambda n, k: (rng.standard_normal((n, k), np.float32) / np.sqrt(k)).astype(np.float16)
    vec = lambda n, s=0.02: (s * rng.standard_normal(n)).astype(np.float32)
    p = "blocks.0."
    return {p + "norm1.weight": 1 + vec(D, 0.1), p + "norm1.bias": vec(D, 0.1), p + "attn.qkv.weight": mat(3 * D, D),
            p + "attn.qkv.bias": vec(3 * D), p + "attn.proj.weight": mat(D, D), p + "attn.proj.bias": vec(D),
            p + "norm2.weight": 1 + vec(D, 0.1), p + "norm2.bias": vec(D, 0.1), p + "mlp.fc1.weight": mat(4 * D, D),
            p + "mlp.fc1.bias": vec(4 * D), p + "mlp.fc2.weight": mat(D, 4 * D), p + "mlp.fc2.bias": vec(D)}


def _put(t, ft, name, a):
    t[name] = a
    ft[name] = 1 if a.dtype == np.float16 else 0


def image_file(D, P=16, C=3, G=4, R=0, pool="token", eps=1e-6, classes=10, pre_norm=False, exact=False, seed=0):
    """A one-block image tower.  exact: integer patch weights in [-2, 2] and conv bias, quarter-integer pos_embed / cls_token / reg_token
    (every embedding sum is exact in f32); otherwise random patch weights, no bias, a zero class token and registers, and pos_embed rows
    of rr.designed_rows, so image 0 (all zero) has rows with the LayerNorm's edge statistics."""
    rng = np.random.default_rng(seed)
    prefix = 0 if pool in gf.PATCH_ONLY_POOLS else 1 + R
    N = G * G + prefix
    t, ft = {}, {}
    if exact:
        _put(t, ft, "patch_embed.proj.weight", rng.integers(-2, 3, (D, C, P, P)).astype(np.float16))
        _put(t, ft, "patch_embed.proj.bias", rng.integers(-4, 5, D).astype(np.float32))
        pos = (rng.integers(-32, 33, (N, D)) / 4).astype(np.float32)
        pre = (rng.integers(-32, 33, (prefix, D)) / 4).astype(np.float32)
    else:
        _put(t, ft, "patch_embed.proj.weight", (rng.standard_normal((D, C, P, P)) / np.sqrt(C * P * P)).astype(np.float16))
        _put(t, ft, "patch_embed.proj.bias", np.zeros(D, np.float32))
        pos = rr.designed_rows(N, D, eps, rng)
        pre = np.zeros((prefix, D), np.float32)
    if prefix:
        _put(t, ft, "cls_token", pre[:1].reshape(1, 1, D))
    if R:
        _put(t, ft, "reg_token", pre[1:].reshape(1, R, D))
    _put(t, ft, "pos_embed", pos.reshape(1, N, D))
    for k, v in _block(D).items():
        _put(t, ft, k, v)
    _put(t, ft, "norm.weight", (1 + 0.2 * rng.standard_normal(D)).astype(np.float32))
    _put(t, ft, "norm.bias", (0.1 * rng.standard_normal(D)).astype(np.float32))
    KH = 2 * D if pool == "cls_patch_mean" else D
    _put(t, ft, "head.weight", (rng.standard_normal((classes, KH)) / np.sqrt(KH)).astype(np.float16))
    _put(t, ft, "head.bias", (0.1 * rng.standard_normal(classes)).astype(np.float32))
    if pre_norm:
        _put(t, ft, "norm_pre.weight", (1 + 0.2 * rng.standard_normal(D)).astype(np.float32))
        _put(t, ft, "norm_pre.bias", (0.1 * rng.standard_normal(D)).astype(np.float32))
    return gf.VitFile(D, 1, D // 64, classes, P, G * P, 1, tensors=t, tensor_ftype=ft, eps=eps, pre_norm=int(pre_norm),
                      activation="gelu_erf", reg_tokens=R, pool=pool)


def images(B, S, C):
    rng = np.random.default_rng(S)
    x = np.stack([AMPS[b % len(AMPS)] * rng.standard_normal((S, S, C)) for b in range(B)]).astype(np.float32)
    return x[..., 0] if C == 1 else x


_cache = {}


def _model(key, build):
    """(VitFile, engine) for `key`, built once; the previous model is released first (the cases of one model run consecutively)."""
    if key not in _cache:
        for k in list(_cache):
            _cache.pop(k)[1].close()
        vf = build()
        _cache[key] = (vf, eng.vit_model_from_tensors(vf, 0, 5))
    return _cache[key]


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    for k in list(_cache):
        _cache.pop(k)[1].close()


def _norm(vf, prefix="norm"):
    return vf.tensors[prefix + ".weight"], vf.tensors[prefix + ".bias"]


def _features(m, imgs, layers, norm, dtype="f32", tokens=True, prelogits=False):
    return eng.vit_features(m, imgs, layers, norm=norm, tokens=tokens, prelogits=prelogits, dtype=DTYPES[dtype])


# ------------------------------------------------------------------------------------------------
# 1. The embedding stage, exact: layer-0 rows equal numpy bit for bit

EMBED_CASES = [(8, 3, 0, "token"), (14, 3, 0, "token"), (16, 3, 0, "token"), (32, 3, 0, "token"), (8, 1, 0, "token"), (16, 1, 0, "token"),
               (16, 3, 0, "cls_patch_mean"), (16, 3, 1, "cls_patch_mean"), (16, 3, 4, "cls_patch_mean"), (16, 3, 16, "cls_patch_mean"),
               (16, 3, 0, "mean")]


@pytest.mark.parametrize("P,C,R,pool", EMBED_CASES, ids=[f"embed-P{p}-C{c}-{pool}-R{r}" for p, c, r, pool in EMBED_CASES])
def test_embedding_exact(P, C, R, pool):
    """Small-integer images, f16-integer patch weights, integer bias, quarter-integer position and prefix rows: every sum is exact, so
    the class and register rows and the patch rows (k = c P^2 + ky P + kx) must equal float64, bit for bit, alone and in a batch of 5."""
    G, D = 3, 64
    vf, m = _model(("embed", P, C, R, pool), lambda: image_file(D, P, C, G, R, pool, exact=True))
    rng = np.random.default_rng(P * 10 + C + R)
    imgs = rng.integers(-3, 4, (5, G * P, G * P, C)).astype(np.float32)
    t = vf.tensors
    prefix = np.concatenate([t[n].reshape(-1, D) for n in ("cls_token", "reg_token") if n in t] or [np.zeros((0, D), np.float32)])
    ref = rr.embed_reference(imgs, t["patch_embed.proj.weight"], t["patch_embed.proj.bias"], t["pos_embed"], prefix, P)
    for B in (1, 5):
        x, _ = _features(m, imgs[:B, ..., 0] if C == 1 else imgs[:B], 0, False)
        rr.check_exact(x, ref[:B], f"B={B}")


# ------------------------------------------------------------------------------------------------
# 2. The final LayerNorm on the features path

LN_CASES = [(D, eps, depth, kind) for D in D_LIST for eps in (1e-6, 1e-5) for depth in (0, 1) for kind in DTYPES]


def _assert_designed(x0, eps):
    """Image 0's layer-0 rows hold what the LayerNorm checks rely on: a row with variance in [eps, 10 eps], and a constant row."""
    var = x0.astype(np.float64).var(-1)
    assert ((var >= eps) & (var <= 10 * eps)).any() and (var == 0).any()


@pytest.mark.parametrize("D,eps,depth,kind", LN_CASES, ids=[f"ln-D{D}-eps{e:g}-depth{k}-{d}" for D, e, k, d in LN_CASES])
def test_final_layernorm(D, eps, depth, kind):
    """Normalised token rows and the token pool's prelogits (row 0) within the LayerNorm bound of float64 applied to the rows observed
    at that depth; the un-normalised ones the RNE of those rows, exactly.  A constant row must come out as norm.bias exactly."""
    vf, m = _model(("ln", D, eps), lambda: image_file(D, eps=eps, seed=D))
    w, b = _norm(vf)
    imgs = images(3, vf.img_size, 3)
    x, _ = _features(m, imgs, depth, False)
    if depth == 0:
        _assert_designed(x[0], eps)
    tok, pre = _features(m, imgs, depth, True, kind, prelogits=True)
    rr.check_layernorm(tok, x, w, b, eps, kind, "tokens")
    rr.check_layernorm(pre[:, 0], x[:, 0], w, b, eps, kind, "prelogits")
    if depth == 0 and kind == "f32":
        const = x[0].astype(np.float64).var(-1) == 0
        assert np.array_equal(tok[0][const], np.broadcast_to(b, tok[0][const].shape))
    raw, rpre = _features(m, imgs, depth, False, kind, prelogits=True)
    rr.check_rounded_rows(raw, x, kind, "raw tokens")
    rr.check_rounded_rows(rpre[:, 0], x[:, 0], kind, "raw prelogits")


# ------------------------------------------------------------------------------------------------
# 3. The pools

def _pool_models():
    out = []
    for i, (R, G) in enumerate(itertools.product([0, 1, 4, 16], [1, 2, 3, 4, 5, 29])):
        out.append(("cls_patch_mean", 2048 if (R, G) == (16, 29) else D_LIST[i % len(D_LIST)], R, G))
    out += [("mean", D, 0, G) for D, G in ((2048, 1), (576, 2), (1088, 3), (320, 29))]
    return out


POOL_CASES = [(pool, D, R, G, kind, norm) for pool, D, R, G in _pool_models() for kind in DTYPES for norm in (True, False)]


@pytest.mark.parametrize("pool,D,R,G,kind,norm", POOL_CASES,
                         ids=[f"pool-{p}-D{D}-R{R}-G{G}-{k}-{'norm' if n else 'raw'}" for p, D, R, G, k, n in POOL_CASES])
def test_pool(pool, D, R, G, kind, norm):
    """The pools' prelogits of 3 images, and of one alone, at depths 0 and 1: un-normalised, bit for bit the kernel's f32 sum order
    rounded once to the output type; normalised, within the LayerNorm and summation bounds of the float64 mean of float64 LayerNorms."""
    vf, m = _model(("pool", pool, D, R, G), lambda: image_file(D, G=G, R=R, pool=pool, seed=D + G + R))
    w, b = _norm(vf)
    first = 0 if pool == "mean" else 1 + R
    imgs = images(3, vf.img_size, 3)
    for depth in (0, 1):
        for batch in (imgs, imgs[1:2]):
            x, _ = _features(m, batch, depth, False)
            _, pre = _features(m, batch, depth, norm, kind, tokens=False, prelogits=True)
            what = f"depth {depth}, B={len(batch)}"
            if norm:
                rr.check_pool_norm(pre[:, 0], x, first, w, b, vf.eps, kind, what)
            else:
                rr.check_pool_raw(pre[:, 0], x, first, kind, what)


# ------------------------------------------------------------------------------------------------
# 3-5. The head's input and the logits through the forward pass

FWD_CASES = [("token", 64, 0, 4, 1), ("token", 576, 0, 4, 3), ("token", 1088, 0, 4, 10), ("token", 2048, 0, 4, 1001),
             ("cls_patch_mean", 320, 4, 3, 10), ("cls_patch_mean", 2048, 16, 5, 1001), ("mean", 1024, 0, 3, 3), ("mean", 512, 0, 29, 10)]


def _check_head(vf, x, a, logits, pool, R):
    """a: the final_ln tap (f16 values, [B][K] or [B][TH][D]) against float64 on x_final; logits against float64 a @ W^T + b."""
    w, b = _norm(vf)
    a16 = a.astype(np.float16)
    if pool == "token":
        rr.check_layernorm(a16, x[:, :a.shape[1]] if a.ndim == 3 else x[:, 0], w, b, vf.eps, "f16", "final_ln")
    else:
        rr.check_pool_norm(a16, x, 0 if pool == "mean" else 1 + R, w, b, vf.eps, "f16", "final_ln")
    ref, bound = rr.logits_bound(a, vf.tensors["head.weight"], vf.tensors["head.bias"])
    rr.check_f32(logits, ref, bound, "logits")


@pytest.mark.parametrize("pool,D,R,G,C", FWD_CASES, ids=[f"forward-{p}-D{D}-R{R}-G{G}-C{c}" for p, D, R, G, c in FWD_CASES])
def test_forward_head(pool, D, R, G, C):
    """vitb200_forward_debug: the final_ln tap within the bounds of float64 applied to the x_final tap, the logits within the f32
    accumulation bound of float64 final_ln @ W^T + b (C % 4 != 0: padded logits rows leave through the 2-D copy)."""
    vf, m = _model(("forward", pool, D, R, G, C), lambda: image_file(D, G=G, R=R, pool=pool, classes=C, seed=C))
    _, logits, taps = eng.vit_predict_debug(m, images(3, vf.img_size, 3), 0, taps=("final_ln", "x_final"))
    _check_head(vf, taps["x_final"], taps["final_ln"], logits, pool, R)


@pytest.mark.parametrize("config", ["vitstr_micro", "vitstr_tiny"], ids=["head25-vitstr_micro", "head25-vitstr_tiny"])
def test_vitstr_25_rows(config):
    """ViTSTR's head over the first 25 rows of each image (rows_per_group / group_stride): the final_ln tap and the logits as above, and
    the features' 25 prelogits rows against the rows at the last depth, normalised in each output type and not."""
    hidden, layers, heads, patch, img = gf.CONFIGS[config]
    classes = gf.NUM_CLASSES[config]
    specs = gf.tensor_specs(hidden, layers, classes, patch, img, 1)
    vf = gf.VitFile(hidden, layers, heads, classes, patch, img, 1, tensors=gf.synth_tensors(hidden, layers, classes, patch, img, 3, in_chans=1),
                    tensor_ftype={n: int(is_mat) for n, _, is_mat in specs})
    m = eng.vit_model_from_tensors(vf, 0, 3, head_tokens=25)
    try:
        imgs = gf.synthetic_gray_images(3, img, seed=4)
        _, logits, taps = eng.vit_predict_debug(m, imgs, 0, taps=("final_ln", "x_final"))
        _check_head(vf, taps["x_final"], taps["final_ln"], logits, "token", 0)
        x, _ = _features(m, imgs, layers, False)
        w, b = _norm(vf)
        for kind in DTYPES:
            _, pre = _features(m, imgs, layers, True, kind, tokens=False, prelogits=True)
            rr.check_layernorm(pre, x[:, :25], w, b, vf.eps, kind, f"prelogits {kind}")
            _, raw = _features(m, imgs, layers, False, kind, tokens=False, prelogits=True)
            rr.check_rounded_rows(raw, x[:, :25], kind, f"raw prelogits {kind}")
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------
# 6. CLIP's pre-norm

@pytest.mark.parametrize("D", D_LIST, ids=[f"prenorm-D{D}" for D in D_LIST])
def test_pre_norm(D):
    """The CLIP tower's layer-0 rows against the float64 LayerNorm (eps 1e-5) of its twin's, the same tensors without norm_pre.  A
    constant row comes out as norm_pre.bias exactly."""
    vf = image_file(D, eps=1e-5, pre_norm=True, seed=D + 1)
    twin = gf.VitFile(**{**vf.__dict__, "pre_norm": 0, "tensors": {k: v for k, v in vf.tensors.items() if not k.startswith("norm_pre.")},
                         "tensor_ftype": {k: v for k, v in vf.tensor_ftype.items() if not k.startswith("norm_pre.")}})
    imgs = images(3, vf.img_size, 3)
    m, mt = eng.vit_model_from_tensors(vf, 0, 3), eng.vit_model_from_tensors(twin, 0, 3)
    try:
        x, _ = _features(mt, imgs, 0, False)
        _assert_designed(x[0], 1e-5)
        y, _ = _features(m, imgs, 0, False)
        w, b = _norm(vf, "norm_pre")
        rr.check_layernorm(y, x, w, b, 1e-5, "f32", "pre-norm")
        const = x[0].astype(np.float64).var(-1) == 0
        assert np.array_equal(y[0][const], np.broadcast_to(b, y[0][const].shape))
    finally:
        m.close()
        mt.close()


# ------------------------------------------------------------------------------------------------
# 7. Text towers

def text_file(D, N, V, pool, eos=7, causal=1, seed=0):
    """A one-block text tower with an identity head (E = D, head.weight = I in f16, bias 0): its embeds are the pooled f16 rows."""
    rng = np.random.default_rng(seed)
    t, ft = {}, {}
    _put(t, ft, "token_embd.weight", rng.standard_normal((V, D)).astype(np.float16))
    _put(t, ft, "pos_embed", (0.5 * rng.standard_normal((1, N, D))).astype(np.float32))
    for k, v in _block(D).items():
        _put(t, ft, k, v)
    _put(t, ft, "norm.weight", (1 + 0.2 * rng.standard_normal(D)).astype(np.float32))
    _put(t, ft, "norm.bias", (0.1 * rng.standard_normal(D)).astype(np.float32))
    _put(t, ft, "head.weight", np.eye(D, dtype=np.float16))
    _put(t, ft, "head.bias", np.zeros(D, np.float32))
    text = {"context": N, "causal": causal, "pool": pool, "eos_token_id": eos, "logit_scale": None, "logit_bias": None}
    return gf.VitFile(D, 1, D // 64, D, 0, 0, 1, tensors=t, tensor_ftype=ft, eps=1e-5, activation="quick_gelu", text=text)


TOKEN_CASES = [(1, 1), (1000, 2), (1000, 31), (1000, 32), (1000, 33), (1000, 77), (1, 77), (1000, 224)]


@pytest.mark.parametrize("V,N", TOKEN_CASES, ids=[f"token_embed-V{V}-N{N}" for V, N in TOKEN_CASES])
def test_token_embed_exact(V, N):
    """Layer-0 token rows equal f32(f16(tok[id])) + pos[t] in numpy f32, bit for bit, with ids 0 and V - 1 present."""
    vf = text_file(64, N, V, "last", seed=N)
    m = eng.vit_model_from_tensors(vf, 0, 3)
    try:
        ids = np.random.default_rng(N).integers(0, V, (3, N))
        ids[0, 0], ids[2, -1] = 0, V - 1
        _, tok = eng.vit_encode_text(m, ids, layers=0, norm=False, tokens=True, embeds=False)
        rr.check_token_embed(tok, ids, vf.tensors["token_embd.weight"], vf.tensors["pos_embed"])
    finally:
        m.close()


def text_ids(pool, B, N, V, eos, rng, shift=0):
    """Sequences whose pooled rows are where the rules differ.  eos: the EOS at 0, in the middle, at N - 1, repeated from position 20
    (padding with EOS), or absent (row 0).  eos_argmax: V - 1 repeated from position 30, 31, 32 or 33 on, as CLIP's padding does.
    Every sequence starts with its own id, holds id 0, and (eos) holds V - 1, which is not the EOS."""
    ids = rng.integers(8, V - 1, (B, N))
    ids[:, 1] = 0
    ids[:, 0] = 8 + np.arange(B)
    if pool == "eos":
        ids[:, 2] = V - 1
    for s in range(B):
        sc = (s + shift) % 5
        if pool == "eos":
            where = {0: [0], 1: [N // 2], 2: [N - 1], 3: list(range(20, N)), 4: []}[sc]
            ids[s, where] = eos
        elif pool == "eos_argmax":
            ids[s, 30 + sc % 4:] = V - 1
    return ids


TEXT_POOL_CASES = [(pool, D, B) for pool in gf.TEXT_POOLS for D, B in ((512, 1), (768, 3), (1024, 4), (1280, 5), (1280, 9))]


@pytest.mark.parametrize("pool,D,B", TEXT_POOL_CASES, ids=[f"text_pool-{p}-D{D}-B{B}" for p, D, B in TEXT_POOL_CASES])
def test_text_pool(pool, D, B):
    """Each sequence's embeds within one f16 rounding of the float64 LayerNorm of the row its rule picks (ties to the first position),
    and outside that of every other candidate row."""
    N, V, eos = 77, 1000, 7
    vf = text_file(D, N, V, pool, eos, seed=D + B)
    m = eng.vit_model_from_tensors(vf, 0, 9)
    try:
        ids = text_ids(pool, B, N, V, eos, np.random.default_rng(B), shift=D // 256)
        emb, x = eng.vit_encode_text(m, ids, layers=1, norm=False, tokens=True, embeds=True)
        w, b = _norm(vf)
        rr.check_text_pool(emb, x, ids, pool, eos, w, b, vf.eps, f"{pool} B={B}")
    finally:
        m.close()
