"""DINOv2 on the GPU (vitb200_arch: the LayerScale residual epilogue, register tokens and the class-plus-patch-mean pool), against the
float64 Hugging Face oracle of tests/dinov2_oracle.py and the emulation of tests/emulation.py.

End to end, every output is held to twice the emulation's own distance from the oracle, measured here on the CPU on the same images
(as tests/test_gpu_clip.py does): the emulation has the engine's roundings and the oracle has none."""
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

# (geometry, with a classifier)
CASES = [("micro", True), ("micro_reg", False), ("s14_reg4", True), ("b14_reg4", True), ("l14", False)]


@pytest.mark.parametrize("K", [768, 3072])
def test_layer_scale_epilogue(K):
    """f32(f32(acc + bias) * gamma) + resid against float64, M not a multiple of 128, gamma from 1e-6 to 10; K = 768 runs the 5-stage
    ring, 3072 (fc2 of D = 768) the 6-stage one.  The bound: the f32 accumulation noise of acc (times gamma) plus the three roundings."""
    M, N = 300, 768
    rng = np.random.default_rng(K)
    A = rng.standard_normal((M, K)).astype(np.float16)
    W = (rng.standard_normal((N, K)) / K ** 0.5).astype(np.float16)
    bias = rng.standard_normal(N).astype(np.float32)
    gamma = np.exp(rng.uniform(np.log(1e-6), np.log(10.0), N)).astype(np.float32)
    resid = rng.standard_normal((M, N)).astype(np.float32)
    out = eng.test_gemm_layer_scale(M, N, K, A, W, bias, gamma, resid)
    acc = A.astype(np.float64) @ W.astype(np.float64).T
    x = acc + bias
    want = x * gamma + resid
    noise = 1e-6 * (np.abs(A).astype(np.float64) @ np.abs(W).astype(np.float64).T + np.abs(bias)) * gamma
    tol = noise + 2.0 ** -23 * (np.abs(x * gamma) * 2 + np.abs(want)) + 1e-30
    err = np.abs(out - want)
    assert (err <= tol).all(), float((err / tol).max())
    # gamma is applied per column, not dropped: the small-gamma columns stay at the residual
    small = gamma < 1e-4
    assert np.allclose(out[:, small], resid[:, small], atol=1e-3)


_built = {}


def _case(geo, classifier, tmp_path_factory):
    key = (geo, classifier)
    if key not in _built:
        d = str(tmp_path_factory.mktemp(f"{geo}_{classifier}"))
        m = do.build_hf(geo, classifier)
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


@pytest.mark.parametrize("geo,classifier", CASES, ids=[f"{g}-{'cls' if c else 'model'}" for g, c in CASES])
def test_end_to_end_against_the_hf_oracle(geo, classifier, tmp_path_factory):
    """logits vs the classifier's logits or pooler_output; prelogits (norm = 1) vs the head's input; tokens (norm = 0) at layers 0, L-1, L
    vs hidden_states; the embed tap vs hidden_states[0]."""
    path, vf, imgs, o, emu_d = _case(geo, classifier, tmp_path_factory)
    L, n, D = vf.num_hidden_layers, imgs.shape[0], vf.hidden_size
    m = eng.vit_model_load(path, 0, n)
    assert (m.layer_scale, m.reg_tokens, m.pool) == (True, vf.reg_tokens, vf.pool) and m.n_tokens == vf.n_tokens
    assert m.arch == {"pre_norm": False, "activation": "gelu_erf"}
    _, _, _, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    got = {"logits": fr.rel_dist(logits, o["logits"])}
    _, pre = eng.vit_features(m, imgs, layers=L, norm=True, tokens=False, prelogits=True)
    assert pre.shape == ((n, 1, 2 * D) if classifier else (n, 1, D))
    got["prelogits"] = fr.rel_dist(pre.reshape(n, -1), o["prelogits"])
    for i in (0, L - 1, L):
        tok, _ = eng.vit_features(m, imgs, layers=i, norm=False)
        assert tok.shape == (n, vf.n_tokens, D)
        got[f"tokens{i}"] = fr.rel_dist(tok, o["hidden_states"][i])
    _, _, taps = eng.vit_predict_debug(m, imgs, 0, taps=("embed",))
    got["embed"] = fr.rel_dist(taps["embed"], o["hidden_states"][0])
    emu_d["embed"] = emu_d["tokens0"]
    m.close()
    print(geo, classifier, {k: f"{got[k].max():.2e} (emulation {emu_d[k].max():.2e})" for k in got})
    bad = {k: (got[k].max(), emu_d[k].max()) for k in got if got[k].max() > 2 * emu_d[k].max()}
    assert not bad, bad


def test_prelogits_forms_agree():
    """The pool kernel's f32, f16 and bf16 outputs, with and without the norm, against the emulation's pool of the same stream."""
    import tempfile
    geo = "micro_reg"
    d = tempfile.mkdtemp()
    path = save_and_convert(do.build_hf(geo, True), d, "dinov2", do.convert_size(geo))
    vf = gf.read_gguf(path)
    imgs = gf.synthetic_images(3, vf.img_size, seed=4)
    m = eng.vit_model_load(path, 0, 3)
    L = vf.num_hidden_layers
    tok, pre = eng.vit_features(m, imgs, layers=L, norm=False, prelogits=True)
    emu = Emulation(vf, fp8=False)
    for norm in (False, True):
        want = emu.prelogits(tok, norm=norm)
        f32 = eng.vit_features(m, imgs, layers=L, norm=norm, tokens=False, prelogits=True)[1].reshape(3, -1)
        assert fr.rel_dist(f32, want).max() <= 2e-6
        f16 = eng.vit_features(m, imgs, layers=L, norm=norm, tokens=False, prelogits=True, dtype=np.float16)[1].reshape(3, -1)
        assert np.array_equal(f16, f32.astype(np.float16))
        bf = eng.vit_features(m, imgs, layers=L, norm=norm, tokens=False, prelogits=True, dtype=eng.BFLOAT16)[1].reshape(3, -1)
        import torch
        assert np.array_equal(bf, torch.from_numpy(f32).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16))
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


def test_every_entry_point_and_the_tensor_path(tmp_path_factory):
    """From tensors == from the file; sharded and device forward == vit_predict; the u8 path == the f32 path on the images it returns."""
    import torch
    path, vf, imgs, _, _ = _case("micro", True, tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3)
    ref = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    mt = eng.vit_model_from_tensors(vf, 0, 3)
    assert (mt.layer_scale, mt.reg_tokens, mt.pool) == (m.layer_scale, m.reg_tokens, m.pool)
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


@pytest.mark.parametrize("geo,classifier", [("micro", True), ("b14_reg4", True)])
def test_fp8_engine_against_the_fp8_emulation(geo, classifier, tmp_path_factory):
    path, vf, imgs, _, _ = _case(geo, classifier, tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3, fp8=True)
    assert m.fp8 and m.layer_scale
    logits = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    m.close()
    d = fr.rel_dist(logits, Emulation(vf).forward(imgs))
    print(f"{geo} FP8: GPU vs emulation {np.array2string(d, precision=4)} (bound {E2E_TOL:.4f})")
    assert d.max() <= E2E_TOL, d
