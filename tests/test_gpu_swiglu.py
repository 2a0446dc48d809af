"""SwiGLU MLPs on the GPU (vitb200_arch.activation = 4, DINOv2 ViT-g): the fc1 epilogue alone in its f16 and e4m3 forms, and whole
models against the float64 Hugging Face oracle of tests/dinov2_oracle.py and the emulation of tests/emulation.py.

End to end, every output is held to twice the emulation's own distance from the oracle, measured here on the CPU on the same images
(the rule of tests/test_gpu_dinov2.py): the emulation has the engine's roundings and the oracle has none."""
import numpy as np
import pytest

from tests.util import pkg, gf
from tests import dinov2_oracle as do
from tests import fp8_reference as fr
from tests.emulation import Emulation
from tests.hf_oracle import save_and_convert
from tests.test_gpu_fp8 import E2E_TOL

eng = pkg.engine
pytestmark = pytest.mark.gpu

# (F, K): the MLP widths of D = 128 (a partial last group of 64), 384, 1024 (partial), 1536 (ViT-g), and K = 3072 for the 6-stage ring;
# K = 80 and 240 (D = 80 H, H odd) end in a partly zero-filled k-block
HOOK_CASES = [(344, 128), (1024, 384), (2736, 1024), (4096, 1536), (4096, 3072), (344, 80), (1024, 240)]
TAIL = 16  # x1 columns driven to x1 << 0 by their bias


def _silu_bound(x1, x2, e1, e2):
    """|error| of f16(silu(x1) x2) given absolute errors e1, e2 of x1 and x2: |silu'| <= 1.1 carries e1, |silu(x1)| carries e2; the
    ex2 / rcp approximation and the rounding of x1 log2(e) cost (|x1| + 4) 2^-22 of silu relative; then one f16 rounding (2^-11, and
    2^-25 absolute below the normal range)."""
    s = x1 / (1.0 + np.exp(-np.maximum(x1, -700.0)))
    want = s * x2
    return want, 1.1 * e1 * np.abs(x2) + np.abs(s) * e2 + (np.abs(x1) + 4) * 2.0 ** -22 * np.abs(want) + 2.0 ** -11 * np.abs(want) + 2.0 ** -25


def _operands(F, K, seed):
    rng = np.random.default_rng(seed)
    M = 300
    A = rng.standard_normal((M, K)).astype(np.float16)
    W = (rng.standard_normal((2 * F, K)) / K ** 0.5).astype(np.float16)
    bias = rng.standard_normal(2 * F).astype(np.float32)
    bias[:TAIL] = -200.0                                     # x1 << 0: silu(x1) underflows, h = +-0
    return M, A, W, bias


@pytest.mark.parametrize("F,K", HOOK_CASES)
def test_swiglu_epilogue(F, K):
    """f16(silu(x1) x2) against float64, x = A W^T + bias with W in HF's order; M = 300 ends inside a tile."""
    M, A, W, bias = _operands(F, K, F + K)
    out = eng.test_gemm(M, 2 * F, K, eng.EPI_SWIGLU, A, W, bias)
    assert out.shape == (M, F)
    a, w = A.astype(np.float64), W.astype(np.float64)
    x = a @ w.T + bias
    noise = 1e-6 * (np.abs(a) @ np.abs(w).T + np.abs(bias))  # the f32 accumulation noise of x
    want, tol = _silu_bound(x[:, :F], x[:, F:], noise[:, :F], noise[:, F:])
    err = np.abs(out - want)
    assert (err <= tol).all(), float((err / tol).max())
    assert (out[:, :TAIL] == 0).all() and np.isfinite(out).all()


@pytest.mark.parametrize("F,K", [(344, 128), (2736, 1024), (4096, 3072), (344, 80), (2736, 1040)])
def test_swiglu_epilogue_e4m3(F, K):
    """The e4m3 form: A rows quantised as the FP8 LayerNorm does (quantize_rows), W as the FP8 upload does (quantize_tensor, HF's order);
    x = acc (sa sw) + bias.  The accumulation bound is test_gpu_fp8's, 2^-9 of sum_k |a w| (Hopper's e4m3 MMA sums)."""
    M, A, W, bias = _operands(F, K, F + K + 1)
    qa, sa = fr.quantize_rows(A.astype(np.float32))
    qw, sw = fr.quantize_tensor(W)
    out = eng.test_gemm_fp8(M, 2 * F, K, eng.EPI_SWIGLU, qa, sa, qw, sw, bias)
    assert out.shape == (M, F)
    a, w = fr.e4m3_value(qa).astype(np.float64), fr.e4m3_value(qw).astype(np.float64)
    s = (sa * sw).astype(np.float32).astype(np.float64)[:, None]
    x = (a @ w.T) * s + bias
    noise = 2.0 ** -9 * (np.abs(a) @ np.abs(w).T) * s + 2.0 ** -24 * np.abs(bias)
    want, tol = _silu_bound(x[:, :F], x[:, F:], noise[:, :F], noise[:, F:])
    err = np.abs(out - want)
    assert (err <= tol).all(), float((err / tol).max())
    assert (out[:, :TAIL] == 0).all() and np.isfinite(out).all()


# (geometry, with a classifier)
CASES = [("micro", True), ("micro_reg", False), ("s14_reg4", True), ("l14", False), ("g14_reg4", True), ("g14_reg4", False)]
_built = {}


def _case(geo, classifier, tmp_path_factory):
    key = (geo, classifier)
    if key not in _built:
        d = str(tmp_path_factory.mktemp(f"swiglu_{geo}_{classifier}"))
        m = do.build_hf(geo, classifier, swiglu=True)
        path = save_and_convert(m, d, "dinov2", do.convert_size(geo))
        vf = gf.read_gguf(path)
        imgs = gf.synthetic_images(3, vf.img_size, seed=3)
        o = do.hf_outputs(m, imgs)
        emu = Emulation(vf, acc=np.float64, fp8=False)
        L = vf.num_hidden_layers
        x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
        emu_d = {"logits": fr.rel_dist(emu.forward(imgs), o["logits"]), "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["prelogits"])}
        emu_d.update({f"tokens{i}": fr.rel_dist(x[i], o["hidden_states"][i]) for i in x})
        _built[key] = (path, vf, imgs, o, emu_d)
    return _built[key]


def _mlp_dim(vf):
    return vf.tensors["blocks.0.mlp.fc2.weight"].shape[1]


@pytest.mark.parametrize("geo,classifier", CASES, ids=[f"{g}-{'cls' if c else 'model'}" for g, c in CASES])
def test_end_to_end_against_the_hf_oracle(geo, classifier, tmp_path_factory):
    """logits vs the classifier's logits or pooler_output; prelogits (norm = 1) vs the head's input; tokens (norm = 0) at layers 0, L-1, L
    vs hidden_states; the embed tap vs hidden_states[0]."""
    path, vf, imgs, o, emu_d = _case(geo, classifier, tmp_path_factory)
    L, n, D = vf.num_hidden_layers, imgs.shape[0], vf.hidden_size
    m = eng.vit_model_load(path, 0, n)
    assert m.arch == {"pre_norm": False, "activation": "swiglu"} and m.mlp_dim == _mlp_dim(vf) and m.n_tokens == vf.n_tokens
    _, _, _, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    got = {"logits": fr.rel_dist(logits, o["logits"])}
    _, pre = eng.vit_features(m, imgs, layers=L, norm=True, tokens=False, prelogits=True)
    got["prelogits"] = fr.rel_dist(pre.reshape(n, -1), o["prelogits"])
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


@pytest.mark.parametrize("geo", ["micro", "l14"])
def test_h_tap_is_swiglu_of_the_ln2_tap(geo, tmp_path_factory):
    """The engine's h [B][N][F] against silu(x1) x2 in float64 of its own ln2 tap times fc1 (HF's order): checks the in-engine
    interleave of weights and bias directly, partial last group included (F = 344, 2736)."""
    path, vf, imgs, _, _ = _case(geo, geo == "micro", tmp_path_factory)
    F = _mlp_dim(vf)
    m = eng.vit_model_load(path, 0, 3)
    for layer in range(vf.num_hidden_layers):
        _, _, taps = eng.vit_predict_debug(m, imgs, layer, taps=("ln2", "h"))
        assert taps["h"].shape == (3, vf.n_tokens, F)
        w = np.asarray(vf.tensors[f"blocks.{layer}.mlp.fc1.weight"], np.float16).astype(np.float64)
        b = np.asarray(vf.tensors[f"blocks.{layer}.mlp.fc1.bias"], np.float64)
        y = taps["ln2"].reshape(-1, vf.hidden_size).astype(np.float64)
        x = y @ w.T + b
        noise = 1e-6 * (np.abs(y) @ np.abs(w).T + np.abs(b))
        want, tol = _silu_bound(x[:, :F], x[:, F:], noise[:, :F], noise[:, F:])
        err = np.abs(taps["h"].reshape(-1, F) - want)
        assert (err <= tol).all(), (layer, float((err / tol).max()))
    m.close()


def test_launch_count_batch_invariance_and_graphs(tmp_path_factory):
    """3 + 7 L + 3 launches; each image alone -- eager, graph capture, graph replay -- gives its logits and its features in the 3-image
    batch, bit for bit."""
    for geo, classifier in (("micro_reg", False), ("micro", True)):
        p, vf, imgs, _, _ = _case(geo, classifier, tmp_path_factory)
        L = vf.num_hidden_layers
        m = eng.vit_model_load(p, 0, 3)
        l_all = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
        assert m.last_launch_count() == 3 + 7 * L + 3
        f_all = eng.vit_features(m, imgs, layers=L, norm=True, prelogits=True, dtype=np.float16)
        for b in range(3):
            for rep in range(3):
                assert np.array_equal(eng.vit_predict(m, imgs[b:b + 1], 5, want_logits=True)[3][0], l_all[b]), (b, rep)
                assert m.last_launch_count() == 3 + 7 * L + 3
                f = eng.vit_features(m, imgs[b:b + 1], layers=L, norm=True, prelogits=True, dtype=np.float16)
                assert np.array_equal(f[0][0], f_all[0][b]) and np.array_equal(f[1][0], f_all[1][b]), (b, rep)
        m.close()


@pytest.mark.parametrize("fp8", [False, True])
def test_every_entry_point_and_the_tensor_path(fp8, tmp_path_factory):
    """From tensors == from the file; sharded and device forward == vit_predict; the u8 path == the f32 path on the images it returns."""
    import torch
    path, vf, imgs, _, _ = _case("micro", True, tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3, fp8=fp8)
    ref = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    mt = eng.vit_model_from_tensors(vf, 0, 3, fp8=fp8)
    assert mt.arch == m.arch and mt.mlp_dim == m.mlp_dim == _mlp_dim(vf)
    assert np.array_equal(eng.vit_predict(mt, imgs, 5, want_logits=True)[3], ref)
    mt.close()
    assert np.array_equal(eng.vit_predict_sharded([m], imgs, 5)[0], eng.vit_predict(m, imgs, 5)[0])
    d_img = torch.from_numpy(imgs).cuda()
    d_log = torch.empty((3, vf.num_classes), dtype=torch.float32, device="cuda")
    eng._check(eng.lib().vitb200_forward_device(m.handle, d_img.data_ptr(), 3, None, d_log.data_ptr(), None, None, 0, None),
               "vitb200_forward_device")
    eng._check(eng.lib().vitb200_sync(m.handle), "vitb200_sync")
    assert np.array_equal(d_log.cpu().numpy(), ref)
    rng = np.random.default_rng(3)
    u8 = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((97, 131), (56, 56), (70, 61))]
    f32, _, _, _, logits = eng.vit_image_preprocess_predict(m, u8)
    assert np.array_equal(logits, eng.vit_predict(m, f32, 5, want_logits=True)[3])
    tok, pre = eng.vit_features_u8(m, u8, layers=1, norm=True, prelogits=True)
    t2, p2 = eng.vit_features(m, f32, layers=1, norm=True, prelogits=True)
    assert np.array_equal(tok, t2) and np.array_equal(pre, p2)
    m.close()


@pytest.mark.parametrize("geo,classifier", [("micro", True), ("g14_reg4", True)])
def test_fp8_engine_against_the_fp8_emulation(geo, classifier, tmp_path_factory):
    path, vf, imgs, _, _ = _case(geo, classifier, tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3, fp8=True)
    assert m.fp8 and m.arch["activation"] == "swiglu"
    logits = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    m.close()
    d = fr.rel_dist(logits, Emulation(vf).forward(imgs))
    print(f"{geo} FP8: GPU vs emulation {np.array2string(d, precision=4)} (bound {E2E_TOL:.4f})")
    assert d.max() <= E2E_TOL, d
