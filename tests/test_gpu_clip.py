"""CLIP image towers on the GPU (vitb200_arch: the pre-norm and the QuickGELU / erf-GELU fc1 epilogues), against the float64 Hugging
Face oracle of tests/clip_oracle.py and the emulation of tests/emulation.py.

End to end, every output is held to twice the emulation's own distance from the oracle, measured here on the CPU on the same images:
the emulation has the engine's roundings (f16 GEMM operands, the reference's f16 soft-max table) and the oracle has none, so an engine
that computes the emulation's function lands at that distance, and a wrong mapping lands orders of magnitude away (tests/test_clip.py)."""
import numpy as np
import pytest

from tests.util import pkg, gf
from tests import clip_oracle as co
from tests import fp8_reference as fr
from tests.emulation import Emulation
from tests.hf_oracle import save_and_convert
from tests.test_gpu_fp8 import E2E_TOL

eng = pkg.engine
pytestmark = pytest.mark.gpu

CASES = [("micro", "quick_gelu"), ("micro", "gelu_erf"), ("b32", "quick_gelu"), ("l14_336", "quick_gelu")]


def _act64(x, epi):
    x = np.asarray(x, np.float64)
    if epi == eng.EPI_BIAS_GELU_ERF_F16:
        from scipy.special import ndtr
        return x * ndtr(x)
    with np.errstate(over="ignore"):
        return x / (1.0 + np.exp(-1.702 * x))


def _tail_bias(N, rng):
    """Bias with every eighth column far in a tail (up to +-3e4, inside the f16 range) and the rest O(1)."""
    b = rng.standard_normal(N).astype(np.float32)
    far = np.array([-3e4, -1e3, -100, -20, -9, 9, 20, 100, 1e3, 3e4], np.float32)
    b[::8] = far[np.arange(len(b[::8])) % len(far)]
    return b


def _check_epilogue(out, x64, acc_scale, epi):
    """out against f16(act(x)), x in float64: the bound of test_gpu_kernels.py::test_gemm_against_numpy for GELU (one f16 ulp, plus the
    slope times the f32 accumulation noise), the noise taken from the size of the sum rather than of the output, since the tail biases
    make the outputs large.  Far left tails give -0 or a tiny negative value."""
    ref = _act64(x64, epi).astype(np.float32).astype(np.float16).astype(np.float32)
    assert np.isfinite(out).all()
    ulp = np.maximum(np.maximum(np.abs(ref), np.abs(x64) * 2.5), 2.0 ** -14) * 2.0 ** -10
    noise = 2e-5 * np.maximum(1.0, acc_scale)
    assert (np.abs(out - ref) <= ulp * 1.001 + noise).all(), float(np.abs(out - ref).max())
    neg, pos = x64 < -20, x64 > 20
    assert (out[neg] <= 0).all() and (np.abs(out[neg]) <= 1e-6).all()       # -0 or a tiny negative value, never NaN
    assert (out[pos] > 0).all()
    return float((out != ref).mean())


@pytest.mark.parametrize("K", [768, 2048])
@pytest.mark.parametrize("epi", [eng.EPI_BIAS_GELU_ERF_F16, eng.EPI_BIAS_QUICK_GELU_F16])
def test_activation_epilogue_f16(epi, K):
    """K = 768 runs the 5-stage ring, 2048 the 6-stage one (fc1 of D = 2048)."""
    M, N = 300, 512
    rng = np.random.default_rng(K + epi)
    A = rng.standard_normal((M, K)).astype(np.float16)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    bias = _tail_bias(N, rng)
    out = eng.test_gemm(M, N, K, epi, A, W, bias)
    acc = A.astype(np.float64) @ W.astype(np.float64).T
    flips = _check_epilogue(out, acc + bias, np.abs(acc).max(), epi)
    assert flips < 0.02, flips


@pytest.mark.parametrize("K", [768, 2048])
@pytest.mark.parametrize("epi", [eng.EPI_BIAS_GELU_ERF_F16, eng.EPI_BIAS_QUICK_GELU_F16])
def test_activation_epilogue_e4m3(epi, K):
    """x = acc (sa sw) + bias on e4m3 operands.  Hopper's e4m3 MMA adds with fewer than f32's mantissa bits (2^-11 of sum |a w| measured in
    test_gpu_fp8.py), so the noise term is that of the sum of |a w|."""
    M, N = 300, 512
    rng = np.random.default_rng(K * 3 + epi)
    qa, sa = fr.quantize_rows(rng.standard_normal((M, K)).astype(np.float32))
    qw, sw = fr.quantize_tensor((rng.standard_normal((N, K)) * 0.05).astype(np.float16))
    bias = _tail_bias(N, rng)
    out = eng.test_gemm_fp8(M, N, K, epi, qa, sa, qw, sw, bias)
    a, w = fr.e4m3_value(qa).astype(np.float64), fr.e4m3_value(qw).astype(np.float64)
    scale = sa.astype(np.float64)[:, None] * float(sw)
    x64 = (a @ w.T) * scale + bias
    mag = (np.abs(a) @ np.abs(w).T) * scale
    ref = _act64(x64, epi).astype(np.float32).astype(np.float16).astype(np.float32)
    assert np.isfinite(out).all()
    ulp = np.maximum(np.maximum(np.abs(ref), np.abs(x64) * 2.5), 2.0 ** -14) * 2.0 ** -10
    assert (np.abs(out - ref) <= ulp * 1.001 + 1.2 * 2.0 ** -10 * mag + 2e-5).all(), float(np.abs(out - ref).max())
    neg, pos = x64 < -20, x64 > 20
    assert (out[neg] <= 0).all() and (np.abs(out[neg]) <= 1e-6).all()
    assert (out[pos] > 0).all()


_built = {}


def _case(geo, act, tmp_path_factory):
    """HF tower -> GGUF, 3 images, the oracle's outputs and the emulation's distances to them (computed once per case)."""
    key = (geo, act)
    if key not in _built:
        d = str(tmp_path_factory.mktemp(f"{geo}_{act}"))
        m = co.build_hf(geo, act)
        path = save_and_convert(m, d, "clip")
        vf = gf.read_gguf(path)
        imgs = gf.synthetic_images(3, vf.img_size, seed=3)
        o = co.hf_outputs(m, imgs)
        emu = Emulation(vf, acc=np.float64, fp8=False)
        L = vf.num_hidden_layers
        x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
        emu_d = {"logits": fr.rel_dist(emu.forward(imgs), o["image_embeds"]),
                 "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["pooler_output"])}
        emu_d.update({f"tokens{i}": fr.rel_dist(x[i], o["hidden_states"][i]) for i in x})
        _built[key] = (path, vf, imgs, o, emu_d)
    return _built[key]


@pytest.mark.parametrize("geo,act", CASES, ids=[f"{g}-{a}" for g, a in CASES])
def test_end_to_end_against_the_hf_oracle(geo, act, tmp_path_factory):
    """logits vs image_embeds; features prelogits (norm = 1) vs pooler_output; features tokens (norm = 0) at layers 0, L-1, L vs
    hidden_states; the embed tap vs hidden_states[0].  l14_336 has 577 tokens, so the mma.sync attention runs."""
    path, vf, imgs, o, emu_d = _case(geo, act, tmp_path_factory)
    L, n = vf.num_hidden_layers, imgs.shape[0]
    m = eng.vit_model_load(path, 0, n)
    assert m.arch == {"pre_norm": True, "activation": act}
    _, _, _, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    got = {"logits": fr.rel_dist(logits, o["image_embeds"])}
    _, pre = eng.vit_features(m, imgs, layers=L, norm=True, tokens=False, prelogits=True)
    got["prelogits"] = fr.rel_dist(pre.reshape(n, -1), o["pooler_output"])
    for i in (0, L - 1, L):
        tok, _ = eng.vit_features(m, imgs, layers=i, norm=False)
        got[f"tokens{i}"] = fr.rel_dist(tok, o["hidden_states"][i])
    _, _, taps = eng.vit_predict_debug(m, imgs, 0, taps=("embed",))
    got["embed"] = fr.rel_dist(taps["embed"], o["hidden_states"][0])
    emu_d["embed"] = emu_d["tokens0"]
    m.close()
    print(geo, act, {k: f"{got[k].max():.2e} (emulation {emu_d[k].max():.2e})" for k in got})
    bad = {k: (got[k].max(), emu_d[k].max()) for k in got if got[k].max() > 2 * emu_d[k].max()}
    assert not bad, bad
    # and against the f16 emulation in f32, as test_gpu_geometry.py holds the logits to the restatement
    emu32 = Emulation(vf, fp8=False).forward(imgs)
    d32 = fr.rel_dist(logits, emu32)
    print(f"{geo} {act}: GPU vs f16 emulation {np.array2string(d32, precision=6)}")
    assert d32.max() <= (1.5e-3 if vf.n_tokens <= 224 else 2e-3), d32


def test_launch_count_batch_invariance_and_graphs(tmp_path_factory):
    """3 + 7 L + 4 launches; each image alone -- eager, graph capture, graph replay -- gives its logits in the 3-image batch, bit for bit,
    and the same for the LLaVA features (layers = L - 1, norm = 0, f16)."""
    path, vf, imgs, _, _ = _case("micro", "quick_gelu", tmp_path_factory)
    L = vf.num_hidden_layers
    m = eng.vit_model_load(path, 0, 3)
    l_all = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    assert m.last_launch_count() == 3 + 7 * L + 4
    f_all = eng.vit_features(m, imgs, layers=L - 1, norm=False, dtype=np.float16)[0]
    for b in range(3):
        for rep in range(3):
            assert np.array_equal(eng.vit_predict(m, imgs[b:b + 1], 5, want_logits=True)[3][0], l_all[b]), (b, rep)
            assert m.last_launch_count() == 3 + 7 * L + 4
            f = eng.vit_features(m, imgs[b:b + 1], layers=L - 1, norm=False, dtype=np.float16)[0]
            assert np.array_equal(f[0], f_all[b]), (b, rep)
    m.close()


def test_every_entry_point_and_the_tensor_path(tmp_path_factory):
    """From tensors == from the file; the u8 path == the f32 path on the images it returns; sharded and device forward == vit_predict."""
    import torch
    path, vf, imgs, _, _ = _case("micro", "gelu_erf", tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3)
    ref = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    mt = eng.vit_model_from_tensors(vf, 0, 3)
    assert mt.arch == m.arch and np.array_equal(eng.vit_predict(mt, imgs, 5, want_logits=True)[3], ref)
    mt.close()
    probs = eng.vit_predict_sharded([m], imgs, 5)[0]
    assert np.array_equal(probs, eng.vit_predict(m, imgs, 5)[0])
    d_img = torch.from_numpy(imgs).cuda()
    d_log = torch.empty((3, vf.num_classes), dtype=torch.float32, device="cuda")
    eng._check(eng.lib().vitb200_forward_device(m.handle, d_img.data_ptr(), 3, None, d_log.data_ptr(), None, None, 0, None),
               "vitb200_forward_device")
    eng._check(eng.lib().vitb200_sync(m.handle), "vitb200_sync")
    assert np.array_equal(d_log.cpu().numpy(), ref)
    rng = np.random.default_rng(3)
    u8 = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((97, 131), (64, 64), (70, 61))]
    f32, _, _, _, logits = eng.vit_image_preprocess_predict(m, u8)
    assert np.array_equal(logits, eng.vit_predict(m, f32, 5, want_logits=True)[3])
    tok = eng.vit_features_u8(m, u8, layers=1, norm=False)[0]
    assert np.array_equal(tok, eng.vit_features(m, f32, layers=1, norm=False)[0])
    m.close()


@pytest.mark.parametrize("geo,act", [("micro", "quick_gelu"), ("micro", "gelu_erf"), ("l14_336", "quick_gelu")])
def test_fp8_engine_against_the_fp8_emulation(geo, act, tmp_path_factory):
    path, vf, imgs, _, _ = _case(geo, act, tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3, fp8=True)
    assert m.fp8 and m.arch["pre_norm"]
    logits = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    m.close()
    d = fr.rel_dist(logits, Emulation(vf).forward(imgs))
    print(f"{geo} {act} FP8: GPU vs emulation {np.array2string(d, precision=4)} (bound {E2E_TOL:.4f})")
    assert d.max() <= E2E_TOL, d
