"""Encoder features (vitb200_features*): the residual stream after any block and the pooled pre-logits rows, checked against the C
restatement (same tolerances as the per-layer taps of test_gpu_forward.py) and bit for bit against the engine's own debug taps."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.util import pkg, gf, model_path
from oracle import restatement as rs

eng = pkg.engine
pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def bf16_bits(x):
    """f32 -> bf16 bit patterns, round to nearest even (finite values)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def layernorm64(x, w, b, eps=1e-6):
    x = x.astype(np.float64)
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * w + b


def final_ln_tap(m, imgs):
    """The head GEMM's A operand (the `final_ln` debug tap, f16 widened), [B][head_tokens][D]; sized for ViTSTR's 25 rows as well."""
    imgs = np.ascontiguousarray(imgs, np.float32)
    B = imgs.shape[0]
    probs = np.empty((B, m.head_tokens, m.num_classes), np.float32)
    logits = np.empty_like(probs)
    out = np.zeros((B, m.head_tokens, m.hidden_size), np.float32)
    tp = eng.Taps()
    tp.layer = 0
    tp.final_ln = out.ctypes.data
    eng._check(eng.lib().vitb200_forward_debug(m.handle, imgs.ctypes.data, B, probs.ctypes.data, logits.ctypes.data, C.byref(tp)),
               "vitb200_forward_debug")
    return out


@pytest.mark.parametrize("cfg", ["micro", "tiny", "large384x2", "d1536"])   # d1536: the row-per-warp kernel at 12 of 16 float4 per lane
def test_features_match_restatement(cfg):
    path = model_path(cfg, "f16")
    vf = gf.read(path)
    om = rs.OracleModel(vf, gf.tensor_specs)
    rs.set_threads(8)
    L = vf.num_hidden_layers
    nw = np.asarray(vf.tensors["norm.weight"], np.float64).reshape(-1)
    nb = np.asarray(vf.tensors["norm.bias"], np.float64).reshape(-1)
    imgs = gf.synthetic_images(2, vf.img_size, seed=7)
    m = eng.vit_model_load(path, 0, 2)
    for layers in sorted({0, 1, L // 2, L}):
        raw, _ = eng.vit_features(m, imgs, layers, norm=False)
        normed, _ = eng.vit_features(m, imgs, layers, norm=True)
        tap, tol = ("embed", 1e-5) if layers == 0 else ("x2", 2e-3)
        for b in range(2):
            r = om.forward(imgs[b], max(layers - 1, 0), (tap,))[2][tap]
            assert np.abs(raw[b] - r).max() <= tol * np.abs(r).max(), (layers, np.abs(raw[b] - r).max(), np.abs(r).max())
            want = layernorm64(r, nw, nb)
            assert np.abs(normed[b] - want).max() <= 3e-3 * np.abs(want).max(), (layers, np.abs(normed[b] - want).max())
    m.close()


def test_features_equal_the_engine_taps():
    m = eng.vit_model_load(model_path("tiny", "f16"), 0, 4)
    L = m.hparams.num_hidden_layers
    imgs = gf.synthetic_images(3, m.img_size, seed=13)
    for layers in (0, 1, 7, L):
        tok, _ = eng.vit_features(m, imgs, layers, norm=False)
        taps = eng.vit_predict_debug(m, imgs, max(layers - 1, 0), taps=("embed", "x2"))[2]
        assert np.array_equal(tok, taps["embed"] if layers == 0 else taps["x2"]), layers
    m.close()


@pytest.mark.parametrize("cfg,head_tokens", [("tiny", 1), ("vitstr_tiny", 25)])
def test_prelogits_are_the_head_input(cfg, head_tokens):
    m = eng.vit_model_load(model_path(cfg, "f16"), 0, 4, head_tokens=head_tokens)
    imgs = (gf.synthetic_images if m.in_chans == 3 else gf.synthetic_gray_images)(3, m.img_size, seed=14)
    _, pre16 = eng.vit_features(m, imgs, tokens=False, prelogits=True, dtype=np.float16)
    assert pre16.shape == (3, head_tokens, m.hidden_size)
    assert np.array_equal(pre16.astype(np.float32), final_ln_tap(m, imgs))
    tok, pre = eng.vit_features(m, imgs, prelogits=True)
    assert np.array_equal(pre, tok[:, :head_tokens])
    m.close()


def _check_16_bit_outputs_are_the_f32_output_rounded(cfg):
    m = eng.vit_model_load(model_path(cfg, "f16"), 0, 4)
    L = m.hparams.num_hidden_layers
    imgs = gf.synthetic_images(3, m.img_size, seed=15)
    for layers in (0, L - 1, L):
        for norm in (False, True):
            t32, p32 = eng.vit_features(m, imgs, layers, norm, prelogits=True)
            t16, p16 = eng.vit_features(m, imgs, layers, norm, prelogits=True, dtype=np.float16)
            tbf, pbf = eng.vit_features(m, imgs, layers, norm, prelogits=True, dtype=eng.BFLOAT16)
            assert t16.dtype == np.float16 and tbf.dtype == np.uint16
            assert np.array_equal(t16.view(np.uint16), t32.astype(np.float16).view(np.uint16)), (layers, norm)
            assert np.array_equal(p16.view(np.uint16), p32.astype(np.float16).view(np.uint16)), (layers, norm)
            assert np.array_equal(tbf, bf16_bits(t32)) and np.array_equal(pbf, bf16_bits(p32)), (layers, norm)
    m.close()


def test_16_bit_outputs_are_the_f32_output_rounded():
    _check_16_bit_outputs_are_the_f32_output_rounded("tiny")


def test_16_bit_outputs_of_the_widest_layernorm_are_the_f32_output_rounded():
    """d1536: the f16 and bf16 forms of the row-per-warp kernel at 16 float4 per lane (1024 < D <= 2048)."""
    _check_16_bit_outputs_are_the_f32_output_rounded("d1536")


def test_batch_invariance_and_graph_replay():
    """An image's features do not depend on its batch mates, its position or the batch size (48 images = 9456 tokens: the eager
    path; 1 and 3 images: the CUDA-graph path), and replayed graphs return what the eager call returned."""
    import torch
    m = eng.vit_model_load(model_path("tiny", "f16"), 0, 48)
    L = m.hparams.num_hidden_layers
    imgs = gf.synthetic_images(48, m.img_size, seed=16)
    args = dict(layers=L - 1, norm=True, prelogits=True)
    t_all, p_all = eng.vit_features(m, imgs, **args)
    for sl in (slice(0, 1), slice(47, 48), slice(20, 23), slice(45, 48)):
        t, p = eng.vit_features(m, imgs[sl], **args)
        assert np.array_equal(t, t_all[sl]) and np.array_equal(p, p_all[sl]), sl
    # host entry: two input slots alternate, so six calls are eager, capture and replay for each slot
    for rep in range(6):
        t, p = eng.vit_features(m, imgs[5:8], **args)
        assert np.array_equal(t, t_all[5:8]) and np.array_equal(p, p_all[5:8]), rep
    # device entry on a caller stream: eager, capture, replay
    d_img = torch.from_numpy(np.ascontiguousarray(imgs[5:8])).cuda()
    d_tok = torch.empty((3, m.n_tokens, m.hidden_size), dtype=torch.float16, device="cuda")
    stream = torch.cuda.Stream()
    req = eng.FeaturesReq(L - 1, 1, 1)
    counts = []
    for rep in range(3):
        d_tok.zero_()
        torch.cuda.synchronize()
        eng._check(eng.lib().vitb200_features_device(m.handle, d_img.data_ptr(), 3, C.byref(req), d_tok.data_ptr(), None, stream.cuda_stream),
                   "vitb200_features_device")
        stream.synchronize()
        counts.append(m.last_launch_count())
        assert np.array_equal(d_tok.cpu().numpy(), t_all[5:8].astype(np.float16)), rep
    assert counts[0] == counts[1] == counts[2] > 0
    m.close()


def test_u8_features_equal_the_features_of_the_preprocessed_images():
    m = eng.vit_model_load(model_path("tiny", "f16"), 0, 4)
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((300, 280), (224, 224), (97, 131))]
    for bilinear in (False, True):
        f32 = eng.vit_image_preprocess_predict(m, imgs, bilinear=bilinear, predict=False)[0]
        for layers, norm, dtype in ((None, True, np.float32), (3, False, np.float16), (0, False, np.float32)):
            got = eng.vit_features_u8(m, imgs, bilinear, layers, norm, prelogits=True, dtype=dtype)
            want = eng.vit_features(m, f32, layers, norm, prelogits=True, dtype=dtype)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (bilinear, layers, norm)
    m.close()


def test_early_exit_launches_fewer_kernels():
    for cfg in ("micro", "tiny"):
        m = eng.vit_model_load(model_path(cfg, "f16"), 0, 2)
        imgs = gf.synthetic_images(2, m.img_size, seed=17)
        counts = []
        for layers in range(m.hparams.num_hidden_layers + 1):
            eng.vit_features(m, imgs, layers, norm=True)
            counts.append(m.last_launch_count())
        assert all(a < b for a, b in zip(counts, counts[1:])), counts
        eng.vit_features(m, imgs, 0, norm=False)  # a plain copy of the residual stream: no kernel after the embeddings
        assert m.last_launch_count() == counts[0] - 1
        m.close()


def test_rejected_requests_leave_the_engine_intact():
    g = np.load(os.path.join(GOLD, "tiny_f16.npz"))
    m = eng.vit_model_load(model_path("tiny", "f16"), 0, 4)
    L = m.hparams.num_hidden_layers
    imgs = gf.synthetic_images(int(g["n_images"]), m.img_size, seed=int(g["image_seed"]))
    want = eng.vit_predict(m, imgs, 5, want_logits=True)
    assert np.abs(want[3] - g["logits"]).max() <= 1.25e-3 * np.abs(g["logits"]).max()
    lib = eng.lib()
    x = np.zeros((1, m.img_size, m.img_size, 3), np.float32)
    out = np.zeros((1, m.n_tokens, m.hidden_size), np.float32)
    for layers, dtype, tok, batch, what in ((-1, 0, out, 1, "layers"), (L + 1, 0, out, 1, "layers"), (L, 3, out, 1, "dtype"),
                                            (L, 0, None, 1, "NULL"), (L, 0, out, 5, "batch"), (L, 0, out, 0, "batch")):
        req = eng.FeaturesReq(layers, 1, dtype)
        assert lib.vitb200_features(m.handle, x.ctypes.data, batch, C.byref(req), tok.ctypes.data if tok is not None else None, None) != 0
        assert what in lib.vitb200_last_error().decode()
    with pytest.raises(ValueError):
        eng.vit_features(m, x, dtype=np.int8)
    got = eng.vit_predict(m, imgs, 5, want_logits=True)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    m.close()

    s = eng.vit_model_load(model_path("vitstr_tiny", "f16"), 0, 2, head_tokens=25)
    gray = gf.synthetic_gray_images(2, s.img_size, seed=18)
    want = eng.vit_predict(s, gray, 5, want_logits=True)
    with pytest.raises(eng.VitB200Error) as ei:
        eng.vit_features_u8(s, [np.zeros((40, 40, 3), np.uint8)])
    assert "1-channel" in str(ei.value)
    got = eng.vit_predict(s, gray, 5, want_logits=True)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    s.close()


def test_classification_is_undisturbed_by_features_calls():
    """vit_predict before and after a sequence of features calls on the same engine is bit-identical, and features from an engine
    that also classifies match those of an engine that only runs features."""
    m = eng.vit_model_load(model_path("micro", "f16"), 0, 5)
    ref = eng.vit_model_load(model_path("micro", "f16"), 0, 5)
    imgs = gf.synthetic_images(5, m.img_size, seed=19)
    want = eng.vit_predict(m, imgs, 5, want_logits=True)
    for layers, norm, dtype in ((1, True, np.float32), (0, False, np.float16), (2, False, np.float32), (1, False, eng.BFLOAT16), (2, True, np.float16)):
        for rep in range(3):
            got = eng.vit_features(m, imgs[:3], layers, norm, prelogits=True, dtype=dtype)
            exp = eng.vit_features(ref, imgs[:3], layers, norm, prelogits=True, dtype=dtype)
            assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (layers, norm, rep)
        after = eng.vit_predict(m, imgs, 5, want_logits=True)
        assert all(np.array_equal(a, b) for a, b in zip(after, want)), (layers, norm)
    m.close()
    ref.close()
