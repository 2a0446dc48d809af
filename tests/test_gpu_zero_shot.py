"""Zero-shot heads on the GPU (vitb200_set_zero_shot): the similarity and top-k kernels against float64, tiny CLIP and SigLIP models
against Hugging Face's logits_per_image, every classification entry point against vitb200_forward, setting, replacing and clearing a head
around cached CUDA graphs, image independence and the launch count, and the setter's refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.util import pkg, gf
from tests import text_oracle as to
from tests.test_gpu_text import _ids

eng = pkg.engine
pytestmark = pytest.mark.gpu

U = 2.0 ** -24
# (logit_scale, logit_bias, probs): CLIP's trained scale of 100 without a bias, SigLIP's initial scale and bias
MODES = [(float(np.log(100.0)), None, "softmax"), (float(np.log(10.0)), -10.0, "sigmoid")]


def _score_bound(E, s, b):
    return 4 * E * U * s + 2 * U * abs(b or 0.0)


def _reference(x, T, logit_scale, logit_bias):
    """float64 scores with the engine's f32 scale."""
    s = float(np.float32(np.exp(logit_scale)))
    return s, eng.zero_shot_logits(x, T, np.log(s), logit_bias)


def _sigmoid64(z):
    z = np.asarray(z, np.float64)
    return np.where(z >= 0, 1 / (1 + np.exp(-np.abs(z))), np.exp(-np.abs(z)) / (1 + np.exp(-np.abs(z))))


@pytest.mark.parametrize("C_", [1, 3, 1000, 57856, 57857])
@pytest.mark.parametrize("E", [64, 512, 768, 1280])
@pytest.mark.parametrize("rows", [1, 37, 256])
def test_hook_against_float64(rows, E, C_):
    """Scores within 4 E 2^-24 s + 2^-23 |b| of float64; CLIP's probabilities and top-k bit for bit those of the soft-max kernel on the same
    scores; sigmoid probabilities within 2^-22 relative (2^-126 absolute below the normal range); top-k ids a stable sort by score (by
    probability for the soft-max, whose f16 exponentials can tie distinct scores); 57 856 and 57 857 classes sit on each side of the
    soft-max's switch to a global working row."""
    rng = np.random.default_rng(rows * 7 + E + C_)
    x = rng.standard_normal((rows, E)).astype(np.float32)
    T = rng.standard_normal((C_, E)).astype(np.float32)
    if C_ >= 6:
        T[5] = T[2] * 4  # equal scores after normalisation: the lower id comes first
    for i, (ls, lb, mode) in enumerate(MODES):
        k = [0, 5, 16][(i + rows + C_) % 3] if C_ > 16 else 16 if i else 5  # k > C with 1 and 3 classes
        probs, lg, idx, val = eng.test_zero_shot(x, T, ls, lb, mode, k)
        s, ref = _reference(x, T, ls, lb)
        err = np.abs(lg - ref).max()
        assert err <= _score_bound(E, s, lb), (mode, err, _score_bound(E, s, lb))
        if C_ >= 6:
            assert np.array_equal(lg[:, 5], lg[:, 2])
        if mode == "softmax":
            p_ref, i_ref, v_ref = eng.test_softmax_topk(lg, k)
            assert np.array_equal(probs, p_ref) and np.array_equal(idx, i_ref) and np.array_equal(val, v_ref)
            key = probs
        else:
            p64 = _sigmoid64(lg)
            assert (np.abs(probs - p64) <= 2.0 ** -22 * p64 + 2.0 ** -126).all()
            key = lg
        if k:
            order = np.argsort(-key, axis=1, kind="stable")[:, :min(k, C_)]
            assert np.array_equal(idx[:, :min(k, C_)], order)
            assert np.array_equal(val[:, :min(k, C_)], np.take_along_axis(probs, order, 1))
            assert (idx[:, C_:] == -1).all() and (val[:, C_:] == 0).all()


def test_hook_nan_rows_and_refusals():
    """A NaN head row gives NaN scores and ids of -1 in both modes while its neighbours keep their bits; a row of zeros is NaN (its norm is
    0); the hook refuses what the setter refuses."""
    rng = np.random.default_rng(1)
    x = rng.standard_normal((4, 64)).astype(np.float32)
    T = rng.standard_normal((10, 64)).astype(np.float32)
    for ls, lb, mode in MODES:
        clean = eng.test_zero_shot(x, T, ls, lb, mode, 3)
        bad = x.copy()
        bad[1, 7] = np.nan
        bad[2] = 0
        got = eng.test_zero_shot(bad, T, ls, lb, mode, 3)
        for r in (1, 2):
            assert np.isnan(got[1][r]).all() and (got[2][r] == -1).all() and (got[3][r] == 0).all()
        for out, ref in zip(got, clean):
            assert np.array_equal(out[[0, 3]], ref[[0, 3]])
    with pytest.raises(eng.VitB200Error, match=r"zero_shot.class_embeds row 4 has zero norm"):
        T0 = T.copy()
        T0[4] = 0
        eng.test_zero_shot(x, T0, 1.0)


@pytest.fixture(scope="module")
def towers(tmp_path_factory):
    """family -> (HF model, image engine path, text engine path, ids): tiny CLIPModel and SiglipModel, both towers converted, as in
    tests/test_gpu_text.py::test_zero_shot."""
    import transformers as tr
    from tests.hf_oracle import init_model
    out = {}
    for family in ("clip", "siglip"):
        d = tmp_path_factory.mktemp(family)
        vision = dict(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, image_size=64, patch_size=16,
                      layer_norm_eps=1e-5 if family == "clip" else 1e-6)
        if family == "clip":
            vision["hidden_act"] = "quick_gelu"
            cfg = tr.CLIPConfig(text_config=to.clip_text_config("micro").to_dict(), vision_config=vision, projection_dim=96)
            model = init_model(tr.CLIPModel, cfg, 1, norms=("layer_norm", "layrnorm"), f32=("position_embedding",))
        else:
            vision["hidden_act"] = "gelu_pytorch_tanh"
            cfg = tr.SiglipConfig(text_config=to.siglip_text_config().to_dict(), vision_config=vision)
            cfg._attn_implementation = "eager"
            model = init_model(tr.SiglipModel, cfg, 1, norms=("norm",), f32=("position_embedding", "probe"))
        with torch.no_grad():
            model.logit_scale.fill_(np.log(10.0))
        model.save_pretrained(str(d))
        st, cj = str(d / "model.safetensors"), str(d / "config.json")
        pkg.convert.main([st, str(d / "img.gguf"), "--hf-config", cj])
        pkg.convert.main([st, str(d / "txt.gguf"), "--hf-config", cj, "--text"])
        ids = _ids(family, gf.read_gguf(str(d / "txt.gguf")), B=5)
        out[family] = (model, str(d / "img.gguf"), str(d / "txt.gguf"), ids)
    return out


def _head(towers, family):
    """(text embeds [5, E], text_arch, set_zero_shot keyword arguments)."""
    _, _, txt, ids = towers[family]
    mt = eng.vit_model_load(txt, 0, 8)
    emb, _ = eng.vit_encode_text(mt, ids)
    ta = mt.text_arch
    mt.close()
    kw = dict(logit_scale=ta["logit_scale"], logit_bias=ta["logit_bias"], probs="softmax" if family == "clip" else "sigmoid")
    return emb, ta, kw


@pytest.mark.parametrize("family", ["clip", "siglip"])
def test_against_hugging_face(towers, family):
    """The engine's scores within the f32 bound of zero_shot_logits on its own image and text embeddings, within test_gpu_text's bound of
    HF's float64 logits_per_image with the same arg-max, and its probabilities HF's softmax(dim=1) (within the f16 exponentials' 2^-10
    relative) or sigmoid (2^-22 relative on the same scores)."""
    model, img, _, ids = towers[family]
    emb, ta, kw = _head(towers, family)
    mi = eng.vit_model_load(img, 0, 8)
    imgs = gf.synthetic_images(4, 64, seed=2) * 0.5
    _, _, _, img_emb = eng.vit_predict(mi, imgs, topk=1, want_logits=True)
    mi.set_zero_shot(emb, labels=[f"class {i}" for i in range(len(emb))], **kw)
    assert mi.n_outputs == len(emb) and mi.labels()[3] == "class 3"
    assert mi.zero_shot == {"n_classes": len(emb), "logit_scale": np.float32(ta["logit_scale"]), "logit_bias": ta["logit_bias"],
                            "probs": kw["probs"]}
    probs, idx, val, lg = eng.vit_predict(mi, imgs, topk=5, want_logits=True)
    assert lg.shape == (4, len(emb)) and idx.shape == (4, 5)
    s, host = _reference(img_emb, emb, ta["logit_scale"], ta["logit_bias"])
    assert np.abs(lg - host).max() <= _score_bound(mi.num_classes, s, ta["logit_bias"])
    m = model.double()
    with torch.no_grad():
        out = m(input_ids=torch.from_numpy(ids.astype(np.int64)), pixel_values=torch.from_numpy(imgs.transpose(0, 3, 1, 2).astype(np.float64)))
    ref = out.logits_per_image
    assert np.abs(lg - ref.numpy()).max() <= 2e-2 * np.abs(ref.numpy()).max() + 1e-3
    assert (lg.argmax(1) == ref.numpy().argmax(1)).all()
    if family == "clip":
        hf = torch.softmax(ref, dim=1).numpy()
        assert np.abs(probs - torch.softmax(torch.from_numpy(lg.astype(np.float64)), 1).numpy()).max() <= 2.0 ** -10
        assert np.abs(probs - hf).max() <= 2e-2
    else:
        p64 = _sigmoid64(lg)
        assert (np.abs(probs - p64) <= 2.0 ** -22 * p64).all()
        assert np.abs(probs - torch.sigmoid(ref).numpy()).max() <= 2e-2
    mi.set_zero_shot(None)
    assert mi.n_outputs == mi.num_classes and mi.zero_shot is None
    mi.close()


def _forward_device(m, imgs, k, stream=None):
    d_img = torch.from_numpy(np.ascontiguousarray(imgs, np.float32)).cuda()
    B, n = len(imgs), m.n_outputs
    p, lg = torch.empty(B, n, device="cuda"), torch.empty(B, n, device="cuda")
    i, v = torch.empty(B, k, dtype=torch.int32, device="cuda"), torch.empty(B, k, device="cuda")
    torch.cuda.synchronize()
    eng._check(eng.lib().vitb200_forward_device(m.handle, d_img.data_ptr(), B, p.data_ptr(), lg.data_ptr(), i.data_ptr(), v.data_ptr(), k,
                                                stream), "vitb200_forward_device")
    torch.cuda.synchronize()
    return p.cpu().numpy(), i.cpu().numpy(), v.cpu().numpy(), lg.cpu().numpy()


def _forward_async(m, imgs, k):
    B, n = len(imgs), m.n_outputs
    x = np.ascontiguousarray(imgs, np.float32)
    p, lg = np.empty((B, n), np.float32), np.empty((B, n), np.float32)
    i, v = np.empty((B, k), np.int32), np.empty((B, k), np.float32)
    eng._check(eng.lib().vitb200_forward_async(m.handle, x.ctypes.data, B, p.ctypes.data, lg.ctypes.data, i.ctypes.data, v.ctypes.data, k),
               "vitb200_forward_async")
    eng._check(eng.lib().vitb200_sync(m.handle), "vitb200_sync")
    return p, i, v, lg


def _equal(a, b):
    return all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


@pytest.mark.parametrize("family", ["clip", "siglip"])
def test_every_entry_point(towers, family):
    """vitb200_forward_async, _device (on the engine's stream and on another), _debug, the u8 entry points with an image processor, both
    sharded forms over two engines and the FP8 engine: the same bits as vitb200_forward on the same engine and images."""
    import transformers as tr
    _, img, _, _ = towers[family]
    emb, _, kw = _head(towers, family)
    imgs = gf.synthetic_images(6, 64, seed=5)
    for fp8 in (False, True):
        m = eng.vit_model_load(img, 0, 8, fp8=fp8)
        m.set_zero_shot(emb, **kw)
        ref = eng.vit_predict(m, imgs, topk=4, want_logits=True)
        assert _equal(_forward_async(m, imgs, 4), ref)
        assert _equal(_forward_device(m, imgs, 4), ref)
        other = torch.cuda.Stream()
        assert _equal(_forward_device(m, imgs, 4, other.cuda_stream), ref)
        probs, logits, _ = eng.vit_predict_debug(m, imgs, 0, taps=("final_ln",))
        assert np.array_equal(probs, ref[0]) and np.array_equal(logits, ref[3])
        if fp8:
            m.close()
            continue
        proc = tr.CLIPImageProcessorPil(size={"shortest_edge": 64}, crop_size={"height": 64, "width": 64})
        m.set_image_proc(proc.to_dict())
        rng = np.random.default_rng(3)
        u8 = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((90, 130), (64, 64), (200, 70))]
        f32, probs, idx, val, logits = eng.vit_image_preprocess_predict(m, u8, topk=4)
        assert _equal((probs, idx, val, logits), eng.vit_predict(m, f32, topk=4, want_logits=True))
        arrs, B, ptrs, nx, ny = eng._u8_batch(u8)
        lg = np.empty((B, m.n_outputs), np.float32)
        eng._check(eng.lib().vitb200_forward_u8_async(m.handle, ptrs, nx, ny, B, 0, None, lg.ctypes.data, None, None, 0), "u8_async")
        eng._check(eng.lib().vitb200_sync(m.handle), "vitb200_sync")
        assert np.array_equal(lg, logits)
        m2 = eng.vit_model_load(img, 0, 8)
        m2.set_zero_shot(emb[:3], **kw)
        hs = (C.c_void_p * 2)(m.handle, m2.handle)
        x = np.ascontiguousarray(imgs, np.float32)
        out = np.empty((6, 5), np.float32)
        with pytest.raises(eng.VitB200Error, match=r"engine 1 returns 3 outputs per row and engine 0 returns 5"):
            eng._check(eng.lib().vitb200_forward_sharded(hs, 2, x.ctypes.data, 6, out.ctypes.data, None, None, None, 0), "sharded")
        m2.set_zero_shot(emb, **kw)
        p, i, v = eng.vit_predict_sharded([m, m2], imgs, topk=4)
        assert _equal((p, i, v), ref[:3])
        p2, i2, v2 = np.empty_like(p), np.empty_like(i), np.empty_like(v)
        eng.vit_predict_sharded_async([m, m2], np.ascontiguousarray(imgs, np.float32), p2, i2, v2)
        eng.sync_all([m, m2])
        assert _equal((p2, i2, v2), ref[:3])
        m2.close()
        m.close()


def test_set_replace_clear_around_graphs(towers):
    """At a batch that replays a cached graph (B = 4) and at one that launches eagerly (B * N > 8192 rows): after a clear the outputs are
    the bits of an engine that never had a head; a head replaced between two replayed calls gives the new head's outputs."""
    _, img, _, _ = towers["clip"]
    emb, _, kw = _head(towers, "clip")
    rng = np.random.default_rng(9)
    emb2 = rng.standard_normal((7, emb.shape[1])).astype(np.float32)
    fresh = eng.vit_model_load(img, 0, 512)
    m = eng.vit_model_load(img, 0, 512)
    for B in (4, 490):
        imgs = gf.synthetic_images(B, 64, seed=B)
        plain = eng.vit_predict(fresh, imgs, topk=5, want_logits=True)
        m.set_zero_shot(emb, **kw)
        one = [_forward_device(m, imgs, 5) for _ in range(3)]  # eager, capture, replay
        assert all(_equal(o, one[0]) for o in one)
        m.set_zero_shot(emb2, **kw)
        two = [_forward_device(m, imgs, 5) for _ in range(3)]
        assert two[0][3].shape == (B, 7) and all(_equal(o, two[0]) for o in two)
        solo = eng.test_zero_shot(plain[3], emb2, kw["logit_scale"], None, "softmax", 5)
        assert _equal((solo[0], solo[2], solo[3], solo[1]), two[0])
        m.set_zero_shot(None)
        for _ in range(3):
            assert _equal(eng.vit_predict(m, imgs, topk=5, want_logits=True), plain)
            assert _equal(_forward_device(m, imgs, 5), plain)
    fresh.close()
    m.close()


@pytest.mark.parametrize("family", ["clip", "siglip"])
def test_isolation_and_launch_count(towers, family):
    """An image alone and inside a batch give the same bits; a NaN image gives a NaN row and ids of -1 and leaves its batch mates as they
    were, eagerly and from a replayed graph; a forward with a head launches one kernel more than without."""
    _, img, _, _ = towers[family]
    emb, _, kw = _head(towers, family)
    m = eng.vit_model_load(img, 0, 8)
    imgs = gf.synthetic_images(5, 64, seed=8)
    eng.vit_predict(m, imgs, topk=5)
    base = m.last_launch_count()
    m.set_zero_shot(emb, **kw)
    batch = eng.vit_predict(m, imgs, topk=5, want_logits=True)
    assert m.last_launch_count() == base + 1
    for b in range(5):
        assert _equal([x[0] for x in eng.vit_predict(m, imgs[b:b + 1], topk=5, want_logits=True)], [x[b] for x in batch])
    bad = imgs.copy()
    bad[2, 10, 10, 0] = np.nan
    for _ in range(3):  # eager, capture, replay
        p, i, v, lg = _forward_device(m, bad, 5)
        assert np.isnan(lg[2]).all() and (i[2] == -1).all() and (v[2] == 0).all()
        keep = [0, 1, 3, 4]
        assert _equal((p[keep], i[keep], v[keep], lg[keep]), [x[keep] for x in batch])
        assert m.last_launch_count() == base + 1
    m.close()


def test_refusals_keep_the_previous_head(towers, tmp_path):
    """Each refusal names the field or the row, and the head set before it stays in force; text, ViTSTR and 1-channel engines refuse a head."""
    from tests.util import model_path
    _, img, txt, _ = towers["clip"]
    emb, _, kw = _head(towers, "clip")
    m = eng.vit_model_load(img, 0, 4)
    imgs = gf.synthetic_images(2, 64, seed=1)
    m.set_zero_shot(emb, **kw)
    ref = eng.vit_predict(m, imgs, topk=3, want_logits=True)
    E = m.num_classes

    def raw(T, n, scale=1.0, bias=float("nan"), mode=0):
        T = np.ascontiguousarray(T, np.float32)
        z = eng.ZeroShot(T.ctypes.data, n, scale, bias, mode)
        eng._check(eng.lib().vitb200_set_zero_shot(m.handle, C.byref(z)), "vitb200_set_zero_shot")

    good = np.ones((3, E), np.float32)
    nan_row = good.copy()
    nan_row[1, 4] = np.nan
    inf_row = good.copy()
    inf_row[2, 0] = -np.inf
    zero_row = good.copy()
    zero_row[0] = 0
    cases = [
        (lambda: raw(good, 0), r"zero_shot.n_classes = 0 out of range \(1..1048576\)"),
        (lambda: raw(good, (1 << 20) + 1), r"zero_shot.n_classes = 1048577 out of range"),
        (lambda: raw(nan_row, 3), r"zero_shot.class_embeds\[1\]\[4\] = nan: must be finite"),
        (lambda: raw(inf_row, 3), r"zero_shot.class_embeds\[2\]\[0\] = -inf: must be finite"),
        (lambda: raw(zero_row, 3), r"zero_shot.class_embeds row 0 has zero norm"),
        (lambda: raw(good, 3, scale=float("inf")), r"zero_shot.logit_scale = inf: must be finite"),
        (lambda: raw(good, 3, scale=float("nan")), r"zero_shot.logit_scale = nan: must be finite"),
        (lambda: raw(good, 3, scale=100.0), r"zero_shot.logit_scale = 100: exp\(logit_scale\) overflows f32"),
        (lambda: raw(good, 3, bias=float("inf")), r"zero_shot.logit_bias = inf: must be finite, or NaN for none"),
        (lambda: raw(good, 3, bias=float("-inf")), r"zero_shot.logit_bias = -inf"),
        (lambda: raw(good, 3, mode=2), r"zero_shot.mode = 2: 0 \(soft-max, CLIP\) or 1 \(sigmoid, SigLIP\)"),
        (lambda: raw(good, 3, mode=-1), r"zero_shot.mode = -1"),
    ]
    for call, message in cases:
        with pytest.raises(eng.VitB200Error, match=message):
            call()
        assert m.n_outputs == len(emb)
        assert _equal(eng.vit_predict(m, imgs, topk=3, want_logits=True), ref)
    with pytest.raises(ValueError, match="probs must be one of"):
        m.set_zero_shot(emb, 1.0, probs="tanh")
    with pytest.raises(ValueError, match=r"class_embeds must be \[classes, 96\]"):
        m.set_zero_shot(emb[:, :10], 1.0)
    assert _equal(eng.vit_predict(m, imgs, topk=3, want_logits=True), ref)
    m.close()
    mt = eng.vit_model_load(txt, 0, 2)
    with pytest.raises(eng.VitB200Error, match="vitb200_set_zero_shot: this is a text engine"):
        mt.set_zero_shot(emb, **kw)
    mt.close()
    ms = eng.vit_model_load(model_path("vitstr_micro", "f16"), 0, 2, head_tokens=25)
    with pytest.raises(eng.VitB200Error, match="this model takes 1-channel input"):
        ms.set_zero_shot(np.ones((2, ms.num_classes), np.float32), 1.0)
    ms.close()
    path = str(tmp_path / "g1.gguf")
    gf.write_synthetic(path, "micro", 1, in_chans=1)
    mg = eng.vit_model_load(path, 0, 2)
    with pytest.raises(eng.VitB200Error, match="this model takes 1-channel input"):
        mg.set_zero_shot(np.ones((2, mg.num_classes), np.float32), 1.0)
    mg.close()
    mv = eng.vit_model_load(model_path("micro", "f16"), 0, 2, head_tokens=4)
    with pytest.raises(eng.VitB200Error, match="head_tokens is 4 \\(ViTSTR\\)"):
        mv.set_zero_shot(np.ones((2, mv.num_classes), np.float32), 1.0)
    mv.close()
