"""SigLIP on the GPU (vitb200_arch pools 2 and 3, activation 3): the gelu_pytorch_tanh epilogue and the probe-attention kernel alone, and
end to end against the float64 Hugging Face oracle of tests/siglip_oracle.py and the emulation of tests/emulation.py.

End to end, every output is held to twice the emulation's own distance from the oracle, measured here on the CPU on the same images
(as tests/test_gpu_dinov2.py does): the emulation has the engine's roundings and the oracle has none."""
import numpy as np
import pytest

from tests.util import pkg, gf
from tests import siglip_oracle as so
from tests import fp8_reference as fr
from tests.emulation import Emulation, gelu_pytorch_tanh
from tests.hf_oracle import save_and_convert
from tests.test_gpu_fp8 import E2E_TOL

eng = pkg.engine
pytestmark = pytest.mark.gpu



def _sparse(rng, rows, K, nnz=16):
    """Rows of K values with nnz entries from {+-0.5, +-1, +-2} and zeros elsewhere: every product and every partial sum of a dot
    product of two such rows is exact in f32 (and in the e4m3 tensor cores' accumulator), so x is known exactly."""
    a = np.zeros((rows, K), np.float32)
    for r in range(rows):
        idx = rng.choice(K, nnz, replace=False)
        a[r, idx] = rng.choice([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0], nnz)
    return a


def _epilogue_inputs(K, seed):
    """M x N problem whose x = acc + bias spans the far left tail to the right: exact accumulators, biases from -12 to 6 plus -1e4."""
    M, N = 200, 512
    rng = np.random.default_rng(seed)
    A, W = _sparse(rng, M, K), _sparse(rng, N, K)
    bias = np.linspace(-12.0, 6.0, N).astype(np.float32)
    bias[::37] = -1e4
    return M, N, A, W, bias


def _check_gelu(out, x32):
    """Each output within one f16 ulp of f16(gelu_pytorch_tanh(x)) (x in f32, evaluated in f64); -0 and never NaN in the left tail."""
    want = gelu_pytorch_tanh(x32.astype(np.float64))
    want16 = want.astype(np.float16)
    ulp = np.spacing(np.abs(want16)).astype(np.float64)
    err = np.abs(out.astype(np.float64) - want16.astype(np.float64))
    assert not np.isnan(out).any()
    assert (err <= ulp).all(), float((err / ulp).max())
    tail = x32 < -10.0
    assert tail.any() and (out[tail] == 0).all() and np.signbit(out[tail]).all()


@pytest.mark.parametrize("K", [768, 3072])
def test_gelu_pytorch_tanh_epilogue_f16(K):
    """Epilogue 10 on f16 operands, K = 768 (the 5-stage ring) and 3072 (the 6-stage one), against float64; activation 0's f16
    pre-rounding gives other results on the same inputs."""
    M, N, A, W, bias = _epilogue_inputs(K, K)
    out = eng.test_gemm(M, N, K, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16, A.astype(np.float16), W.astype(np.float16), bias)
    x32 = (A.astype(np.float64) @ W.astype(np.float64).T).astype(np.float32) + bias
    _check_gelu(out, x32)
    table = eng.test_gemm(M, N, K, eng.EPI_BIAS_GELU_F16, A.astype(np.float16), W.astype(np.float16), bias)
    differ = int((table != out).sum())
    print(f"K {K}: {differ} of {out.size} outputs differ from activation 0's (f16-rounded x)")
    assert differ > 0


@pytest.mark.parametrize("K", [768, 3072])
def test_gelu_pytorch_tanh_epilogue_e4m3(K):
    """The same on the e4m3 tensor cores: x = acc (sa sw) + bias with power-of-two scales, so x is exact in f32 too."""
    M, N, A, W, bias = _epilogue_inputs(K, K + 1)
    sa = np.full(M, 0.25, np.float32)
    sw = 0.5
    A8, W8 = fr.e4m3_bits(A), fr.e4m3_bits(W)
    assert np.array_equal(fr.e4m3_value(A8), A) and np.array_equal(fr.e4m3_value(W8), W)
    out = eng.test_gemm_fp8(M, N, K, eng.EPI_BIAS_GELU_PYTORCH_TANH_F16, A8, sa, W8, sw, bias)
    acc = A.astype(np.float64) @ W.astype(np.float64).T
    x32 = (acc * (0.25 * sw)).astype(np.float32) + bias
    _check_gelu(out, x32)
    table = eng.test_gemm_fp8(M, N, K, eng.EPI_BIAS_GELU_F16, A8, sa, W8, sw, bias)
    assert int((table != out).sum()) > 0


# token counts on both sides of the kernel's 32-key passes, up to the engine's 896
POOL_P = [1, 31, 32, 33, 63, 64, 65, 195, 196, 197, 255, 256, 257, 575, 576, 577, 895, 896]


def _pool_ref(q, kv, B, P, H):
    D = H * 64
    kv = kv.astype(np.float64).reshape(B, P, 2, H, 64)
    s = np.einsum("hd,bphd->bhp", q.astype(np.float64).reshape(H, 64), kv[:, :, 0]) / 8.0
    p = np.exp(s - s.max(axis=2, keepdims=True))
    p /= p.sum(axis=2, keepdims=True)
    return np.einsum("bhp,bphd->bhd", p, kv[:, :, 1]).reshape(B, D)


@pytest.mark.parametrize("P", POOL_P)
def test_attention_pool_kernel(P):
    """Random q, k, v against float64 (f16 output: one ulp plus the f32 sums); one-hot scores give the chosen v row bit for bit; equal
    scores give each image's plain mean, so a counted padded key or a neighbour's row fails; NaN / Inf in one image's k or v leaves the
    other images bit-identical."""
    B, H = 3, 2
    D = H * 64
    rng = np.random.default_rng(P)
    q = rng.standard_normal(D).astype(np.float32)
    kv = rng.standard_normal((B * P, 2 * D)).astype(np.float16)
    out = eng.test_attention_pool(q, kv, B, P, H)
    want = _pool_ref(q, kv, B, P, H)
    assert np.abs(out - want).max() <= 2e-3 * np.abs(want).max() + 1e-3, np.abs(out - want).max()
    # one-hot: score 16 * 64 / 8 = 128 for the chosen key, 0 for the rest (exp(-128) is 0 in f32)
    ones = np.ones(D, np.float32)
    hot = np.zeros((B * P, 2 * D), np.float16)
    hot[:, D:] = rng.standard_normal((B * P, D)).astype(np.float16)
    chosen = rng.integers(0, P, B)
    for b in range(B):
        hot[b * P + chosen[b], :D] = 16.0
    got = eng.test_attention_pool(ones, hot, B, P, H)
    for b in range(B):
        assert np.array_equal(got[b], hot[b * P + chosen[b], D:].astype(np.float32)), b
    # uniform: k = 0, image b's values all b + 1 -> exactly b + 1
    uni = np.zeros((B * P, 2 * D), np.float16)
    for b in range(B):
        uni[b * P:(b + 1) * P, D:] = b + 1
    got = eng.test_attention_pool(q, uni, B, P, H)
    assert np.array_equal(got, np.repeat(np.arange(1, B + 1, dtype=np.float32), D).reshape(B, D))
    # non-finite values in image 1's k or v
    for col, val in ((3, np.nan), (D + 5, np.inf), (7, -np.inf)):
        bad = kv.copy()
        bad[P + P // 2, col] = val
        got = eng.test_attention_pool(q, bad, B, P, H)
        assert np.array_equal(got[0], out[0]) and np.array_equal(got[2], out[2]), (col, val)


_built = {}


def _case(geo, classifier, tmp_path_factory):
    key = (geo, classifier)
    if key not in _built:
        d = str(tmp_path_factory.mktemp(f"{geo}_{classifier}"))
        m = so.build_hf(geo, classifier)
        path = save_and_convert(m, d, "siglip")
        vf = gf.read_gguf(path)
        imgs = gf.synthetic_images(3, vf.img_size, seed=3)
        o = so.hf_outputs(m, imgs)
        emu = Emulation(vf, acc=np.float64, fp8=False)
        L = vf.num_hidden_layers
        x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
        emu_d = {"logits": fr.rel_dist(emu.forward(imgs), o["logits"]), "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["prelogits"]),
                 "last_hidden_state": fr.rel_dist(emu.final_ln(x[L]), o["last_hidden_state"])}
        emu_d.update({f"tokens{i}": fr.rel_dist(x[i], o["hidden_states"][i]) for i in x})
        _built[key] = (path, vf, imgs, o, emu_d)
    return _built[key]


CASES = [(g, c) for g in so.GEOMETRIES for c in (False, True)]


@pytest.mark.parametrize("geo,classifier", CASES, ids=[f"{g}-{'cls' if c else 'model'}" for g, c in CASES])
def test_end_to_end_against_the_hf_oracle(geo, classifier, tmp_path_factory):
    """logits vs the classifier's logits or pooler_output; prelogits (norm = 1) vs pooler_output or the token mean; tokens (norm = 0) at
    layers 0, L-1, L vs hidden_states; tokens (norm = 1) vs last_hidden_state; the embed tap vs hidden_states[0]."""
    path, vf, imgs, o, emu_d = _case(geo, classifier, tmp_path_factory)
    L, n, D, P = vf.num_hidden_layers, imgs.shape[0], vf.hidden_size, vf.n_tokens
    m = eng.vit_model_load(path, 0, n)
    assert m.pool == ("mean" if classifier else "map") and m.n_tokens == P == (vf.img_size // 16) ** 2
    assert m.arch == {"pre_norm": False, "activation": "gelu_pytorch_tanh"}
    _, _, _, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    got = {"logits": fr.rel_dist(logits, o["logits"])}
    tok, pre = eng.vit_features(m, imgs, layers=L, norm=True, prelogits=True)
    assert pre.shape == (n, 1, D) and tok.shape == (n, P, D)
    got["prelogits"] = fr.rel_dist(pre.reshape(n, -1), o["prelogits"])
    got["last_hidden_state"] = fr.rel_dist(tok, o["last_hidden_state"])
    for i in (0, L - 1, L):
        tok, _ = eng.vit_features(m, imgs, layers=i, norm=False)
        got[f"tokens{i}"] = fr.rel_dist(tok, o["hidden_states"][i])
    _, _, taps = eng.vit_predict_debug(m, imgs, 0, taps=("embed",))
    got["embed"] = fr.rel_dist(taps["embed"], o["hidden_states"][0])
    emu_d["embed"] = emu_d["tokens0"]
    m.close()
    print(geo, classifier, {k: f"{got[k].max():.2e} (emulation {emu_d[k].max():.2e})" for k in got})
    bad = {k: (got[k].max(), emu_d[k].max()) for k in got if got[k].max() > 2 * emu_d[k].max()}
    assert not bad, bad


def test_prelogits_forms_and_the_norm_requirement(tmp_path_factory):
    """The map head's f16 / bf16 prelogits are its f32 row rounded; the mean pool's with and without the norm match the emulation's
    mean of the same stream; map prelogits without the norm are refused before anything runs."""
    import torch
    for classifier in (False, True):
        path, vf, imgs, _, _ = _case("micro", classifier, tmp_path_factory)
        m = eng.vit_model_load(path, 0, 3)
        L = vf.num_hidden_layers
        for norm in ((True,) if not classifier else (False, True)):
            f32 = eng.vit_features(m, imgs, layers=L, norm=norm, tokens=False, prelogits=True)[1].reshape(3, -1)
            f16 = eng.vit_features(m, imgs, layers=L, norm=norm, tokens=False, prelogits=True, dtype=np.float16)[1].reshape(3, -1)
            assert np.array_equal(f16, f32.astype(np.float16))
            bf = eng.vit_features(m, imgs, layers=L, norm=norm, tokens=False, prelogits=True, dtype=eng.BFLOAT16)[1].reshape(3, -1)
            assert np.array_equal(bf, torch.from_numpy(f32).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16))
            if classifier:
                tok = eng.vit_features(m, imgs, layers=L, norm=False)[0]
                assert fr.rel_dist(f32, Emulation(vf, fp8=False).prelogits(tok, norm=norm)).max() <= 2e-6
        if not classifier:
            launches = m.last_launch_count()
            with pytest.raises(eng.VitB200Error, match="prelogits need norm = 1"):
                eng.vit_features(m, imgs, layers=L, norm=False, prelogits=True)
            assert m.last_launch_count() == launches
            # the head at another depth, and the tokens staged next to it on the host path
            tok, pre = eng.vit_features(m, imgs, layers=1, norm=True, prelogits=True)
            emu = Emulation(vf, fp8=False)
            x1 = emu.encode(imgs, 1)
            assert fr.rel_dist(pre.reshape(3, -1), emu.prelogits(x1)).max() <= 1e-2
            assert fr.rel_dist(tok, emu.final_ln(x1)).max() <= 1e-2
        m.close()


def test_launch_count_batch_invariance_and_graphs(tmp_path_factory):
    """2 + 7 L + 10 launches (map) and 2 + 7 L + 3 (mean); each image alone -- eager, graph capture, graph replay -- gives its logits and
    its features in the 3-image batch, bit for bit."""
    for classifier in (False, True):
        p, vf, imgs, _, _ = _case("micro", classifier, tmp_path_factory)
        L = vf.num_hidden_layers
        want = 2 + 7 * L + (3 if classifier else 10)
        m = eng.vit_model_load(p, 0, 3)
        l_all = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
        assert m.last_launch_count() == want
        f_all = eng.vit_features(m, imgs, layers=L, norm=True, prelogits=True, dtype=np.float16)
        for b in range(3):
            for rep in range(3):
                assert np.array_equal(eng.vit_predict(m, imgs[b:b + 1], 5, want_logits=True)[3][0], l_all[b]), (b, rep)
                assert m.last_launch_count() == want
                f = eng.vit_features(m, imgs[b:b + 1], layers=L, norm=True, prelogits=True, dtype=np.float16)
                assert np.array_equal(f[0][0], f_all[0][b]) and np.array_equal(f[1][0], f_all[1][b]), (b, rep)
        m.close()


def test_profile_kind_8_is_the_pooling_head(tmp_path_factory):
    import ctypes as C
    p, vf, imgs, _, _ = _case("micro", False, tmp_path_factory)
    m = eng.vit_model_load(p, 0, 3)
    L = eng.lib()
    eng._check(L.vitb200_profile_enable(m.handle, 1), "profile")
    eng.vit_predict(m, imgs, 5)
    ms, cnt, fl = C.c_double(), C.c_int(), C.c_double()
    counts = []
    for kind in range(9):
        eng._check(L.vitb200_profile_read(m.handle, kind, C.byref(ms), C.byref(cnt), C.byref(fl)), "profile_read")
        counts.append(cnt.value)
    eng._check(L.vitb200_profile_enable(m.handle, 0), "profile")
    assert counts[8] == 3 and counts[5] == 1           # kv + attention + out_proj, fc1 + fc2, the f16 rounding; the head GEMM
    assert counts[7] == 2 * vf.num_hidden_layers + 2   # the block LayerNorms and the head's two
    with pytest.raises(eng.VitB200Error, match="profile kind 9 out of range"):
        eng._check(L.vitb200_profile_read(m.handle, 9, C.byref(ms), C.byref(cnt), C.byref(fl)), "profile_read")
    m.close()


def test_every_entry_point_and_the_tensor_path(tmp_path_factory):
    """From tensors == from the file; sharded and device forward == vit_predict; the u8 path == the f32 path on the images it returns;
    the device features path == the host one."""
    import torch
    for classifier in (False, True):
        path, vf, imgs, _, _ = _case("micro", classifier, tmp_path_factory)
        m = eng.vit_model_load(path, 0, 3)
        ref = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
        mt = eng.vit_model_from_tensors(vf, 0, 3)
        assert mt.pool == m.pool and mt.n_tokens == m.n_tokens
        assert np.array_equal(eng.vit_predict(mt, imgs, 5, want_logits=True)[3], ref)
        mt.close()
        assert np.array_equal(eng.vit_predict_sharded([m], imgs, 5)[0], eng.vit_predict(m, imgs, 5)[0])
        d_img = torch.from_numpy(imgs).cuda()
        d_log = torch.empty((3, vf.num_classes), dtype=torch.float32, device="cuda")
        eng._check(eng.lib().vitb200_forward_device(m.handle, d_img.data_ptr(), 3, None, d_log.data_ptr(), None, None, 0, None),
                   "vitb200_forward_device")
        d_tok = torch.empty((3, vf.n_tokens, vf.hidden_size), dtype=torch.float32, device="cuda")
        d_pre = torch.empty((3, 1, vf.hidden_size), dtype=torch.float32, device="cuda")
        req = eng.FeaturesReq(vf.num_hidden_layers, 1, 0)
        import ctypes as C
        eng._check(eng.lib().vitb200_features_device(m.handle, d_img.data_ptr(), 3, C.byref(req), d_tok.data_ptr(), d_pre.data_ptr(), None),
                   "vitb200_features_device")
        eng._check(eng.lib().vitb200_sync(m.handle), "vitb200_sync")
        torch.cuda.synchronize()
        assert np.array_equal(d_log.cpu().numpy(), ref)
        tok, pre = eng.vit_features(m, imgs, norm=True, prelogits=True)
        assert np.array_equal(d_tok.cpu().numpy(), tok) and np.array_equal(d_pre.cpu().numpy(), pre)
        rng = np.random.default_rng(3)
        u8 = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((97, 131), (64, 64), (70, 61))]
        f32, _, _, _, logits = eng.vit_image_preprocess_predict(m, u8)
        assert np.array_equal(logits, eng.vit_predict(m, f32, 5, want_logits=True)[3])
        tok, pre = eng.vit_features_u8(m, u8, layers=1, norm=True, prelogits=True)
        t2, p2 = eng.vit_features(m, f32, layers=1, norm=True, prelogits=True)
        assert np.array_equal(tok, t2) and np.array_equal(pre, p2)
        m.close()


def test_a_poisoned_image_leaves_its_batch_mates_alone(tmp_path_factory):
    """One NaN pixel, or every pixel at 1e6, in image 1: images 0 and 2 keep their logits and features bit for bit."""
    for classifier in (False, True):
        path, vf, imgs, _, _ = _case("micro", classifier, tmp_path_factory)
        m = eng.vit_model_load(path, 0, 3)
        clean = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
        ctok, cpre = eng.vit_features(m, imgs, norm=True, prelogits=True)
        for poison in ("nan", "big"):
            bad = imgs.copy()
            if poison == "nan":
                bad[1, 5, 7, 1] = np.nan
            else:
                bad[1] = 1e6
            logits = eng.vit_predict(m, bad, 5, want_logits=True)[3]
            tok, pre = eng.vit_features(m, bad, norm=True, prelogits=True)
            for b in (0, 2):
                assert np.array_equal(logits[b], clean[b]) and np.array_equal(tok[b], ctok[b]) and np.array_equal(pre[b], cpre[b]), (poison, b)
        assert np.array_equal(eng.vit_predict(m, imgs, 5, want_logits=True)[3], clean)
        m.close()


@pytest.mark.parametrize("geo,classifier", [("micro", False), ("b16_224", False), ("l16_384", True)])
def test_fp8_engine_against_the_fp8_emulation(geo, classifier, tmp_path_factory):
    path, vf, imgs, _, _ = _case(geo, classifier, tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3, fp8=True)
    assert m.fp8 and m.pool == ("mean" if classifier else "map")
    logits = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    m.close()
    d = fr.rel_dist(logits, Emulation(vf).forward(imgs))
    print(f"{geo} FP8: GPU vs emulation {np.array2string(d, precision=4)} (bound {E2E_TOL:.4f})")
    assert d.max() <= E2E_TOL, d
