"""Text recognition with ViTSTR models (vitb200_recognize_u8*, vitstr_recognize_u8 / vitstr_preprocess_u8): the extension's grayscale
preprocess bit for bit (live extension, committed fixture, and an exact gray-level emulation), the patch-matrix path against the f32
path, the greedy decode against a numpy decode of the call's own probabilities, the pipeline, the launch count and the rejections."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import ref
from tests import vitstr_reference as vr
from tests.util import pkg, gf, model_path

eng = pkg.engine
pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def recognize(m, imgs, f32=True):
    """vitb200_recognize_u8 with every output: (images_f32 [B,S,S], chars, lengths, scores, probs [B,n,C])."""
    imgs = [np.ascontiguousarray(a, np.uint8) for a in imgs]
    B, S, n = len(imgs), m.img_size, m.head_tokens
    out = (np.empty((B, S, S), np.float32) if f32 else None, np.empty((B, n - 1), np.int32), np.empty(B, np.int32),
           np.empty(B, np.float64), np.empty((B, n, m.num_classes), np.float32))
    ptrs = (C.c_void_p * B)(*[a.ctypes.data for a in imgs])
    nx = (C.c_int * B)(*[a.shape[1] for a in imgs])
    ny = (C.c_int * B)(*[a.shape[0] for a in imgs])
    rc = eng.lib().vitb200_recognize_u8(m.handle, ptrs, nx, ny, B, *[None if a is None else a.ctypes.data for a in out])
    if rc != 0:
        raise eng.VitB200Error(eng.lib().vitb200_last_error().decode())
    return out


def sized_images(S, seed):
    rng = np.random.default_rng(seed)
    sizes = [(2, 2), (5, 17), (97, 3), (700, 50), (40, 1000), (120, 300), (S, S)]  # (height, width)
    imgs = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]
    return imgs + [np.zeros((24, 64, 3), np.uint8), np.full((64, 24, 3), 255, np.uint8)]


def word_crops(n, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, size=(int(rng.integers(24, 129)), int(rng.integers(64, 401)), 3), dtype=np.uint8) for _ in range(n)]


def test_preprocess_matches_the_committed_fixture_bit_for_bit():
    g = np.load(os.path.join(GOLD, "vitstr_preprocess.npz"))
    m = eng.vit_model_load(model_path("vitstr_micro", "f16"), 0, 8, head_tokens=25)
    assert m.img_size == int(g["img_size"])
    imgs, off = [], 0
    for h, w, c in g["shapes"]:
        imgs.append(g["pixels"][off:off + h * w * c].reshape(h, w, c))
        off += h * w * c
    assert off == g["pixels"].size
    assert np.array_equal(eng.vitstr_preprocess_u8(m, imgs), g["images_f32"])
    assert np.array_equal(recognize(m, imgs)[0], g["images_f32"])  # the same pixels when the forward pass and decode follow
    m.close()


@pytest.mark.skipif(not vr.available(), reason="oracle/_ref/libvitstrref.so not shipped")
@pytest.mark.parametrize("cfg", ["vitstr_micro", "vitstr_tiny"])
def test_preprocess_matches_the_live_extension_bit_for_bit(cfg):
    m = eng.vit_model_load(model_path(cfg, "f16"), 0, 9, head_tokens=25)
    imgs = sized_images(m.img_size, seed=5)
    got = eng.vitstr_preprocess_u8(m, imgs)
    for b, im in enumerate(imgs):
        assert np.array_equal(got[b], vr.preprocess(im, m.img_size)), (b, im.shape)
    m.close()


def test_gray_levels_truncate_as_the_extension_does():
    """At scale 1 (an S x S image) u = v = 0, so every output is the gray level of one source pixel -- row / column S-2 for the last
    row / column (the clamp).  Sweeping (v, v, v) over all 256 levels, exactly 75 come out as v - 1 (emulated exactly in rationals)."""
    m = eng.vit_model_load(model_path("vitstr_micro", "f16"), 0, 2, head_tokens=25)
    S = m.img_size
    lv = (np.arange(S * S) % 256).reshape(S, S).astype(np.uint8)
    got = eng.vitstr_preprocess_u8(m, [np.repeat(lv[:, :, None], 3, axis=2)])[0]
    gray = np.array([vr.gray_level(v) for v in range(256)])
    assert sum(gray[v] == v - 1 for v in range(256)) == 75 and (gray[[1, 2, 4, 8, 13]] == [0, 1, 3, 7, 12]).all() and gray[255] == 255
    src = np.minimum(np.arange(S), S - 2)
    g = gray[lv[src][:, src]].astype(np.float32)
    want = (g / np.float32(255) - np.float32(0.5)) * np.float32(2)
    assert np.array_equal(got, want)
    m.close()


@pytest.mark.parametrize("cfg", ["vitstr_micro", "vitstr_tiny"])
def test_patch_matrix_path_equals_the_f32_path(cfg):
    m = eng.vit_model_load(model_path(cfg, "f16"), 0, 6, head_tokens=25)
    f32, chars, lengths, scores, probs = recognize(m, word_crops(6, seed=3))
    assert np.array_equal(probs, eng.vit_predict(m, f32, 5)[0])
    m.close()


def _head_edit(fn):
    def edit(entries):
        for e in entries:
            if e[0] in ("head.weight", "head.bias"):
                e[1] = e[1].copy()
        w = next(e[1] for e in entries if e[0] == "head.weight")
        b = next(e[1] for e in entries if e[0] == "head.bias")
        fn(w, b)
        return entries
    return edit


def _check_decode(m, imgs):
    f32, chars, lengths, scores, probs = recognize(m, imgs)
    want = vr.greedy_decode(probs)
    assert np.array_equal(chars, want[0]) and np.array_equal(lengths, want[1]) and np.array_equal(scores, want[2])
    return chars, lengths, scores, probs


def test_decode_is_exact():
    vf = gf.read(model_path("vitstr_micro", "f16"))
    imgs = word_crops(5, seed=8)
    m = eng.vit_model_from_tensors(vf, max_batch=5, head_tokens=25)
    _check_decode(m, imgs)
    m.close()

    def tie(w, b):  # classes 5 and 9 identical and dominant, [s] never wins: the lower id, every token
        w[9] = w[5]
        b[5] = b[9] = b.max() + 20
        b[1] = b.min() - 30
    m = eng.vit_model_from_tensors(vf, max_batch=5, head_tokens=25, edit=_head_edit(tie))
    chars, lengths, scores, probs = _check_decode(m, imgs)
    assert np.array_equal(probs[:, 1:, 5], probs[:, 1:, 9])  # an exact tie
    assert (chars == 5).all() and (lengths == 24).all() and (scores < 1).all()
    m.close()

    def eos(w, b):  # [s] dominant from token 1: empty strings
        b[1] = b.max() + 30
    m = eng.vit_model_from_tensors(vf, max_batch=5, head_tokens=25, edit=_head_edit(eos))
    chars, lengths, scores, probs = _check_decode(m, imgs)
    assert (chars == -1).all() and (lengths == 0).all() and (scores == 1.0).all()
    texts = eng.vitstr_recognize_u8(m, imgs)[0]
    assert texts is None  # a model built from tensors has no id2label
    m.close()


@pytest.mark.skipif(not ref.vitstr_available(), reason="oracle/_ref/libvitstrref.so not shipped")
def test_recognition_matches_the_live_extension():
    """The extension's preprocess + forward + greedy decode against ours: ids agree wherever the extension's top-2 logit gap exceeds
    2.5x our logit deviation (the criterion of the classifier parity test), scores within the probability tolerance."""
    path = model_path("vitstr_tiny", "f16")
    m = eng.vit_model_load(path, 0, 4, head_tokens=25)
    rm = ref.VitstrRefModel(path)
    imgs = word_crops(4, seed=13)
    texts, scores, chars, lengths, probs = eng.vitstr_recognize_u8(m, imgs, probs=True)
    f32 = eng.vitstr_preprocess_u8(m, imgs)
    logits = eng.vit_predict(m, f32, 5, want_logits=True)[3]
    n_clear = 0
    for b, im in enumerate(imgs):
        g = vr.preprocess(im, m.img_size)
        assert np.array_equal(f32[b], g)
        p_ref, l_ref = rm.predict(g, n_threads=8)
        top2 = np.sort(l_ref, -1)[:, -2:]
        dl = np.abs(logits[b] - l_ref).max(-1)
        clear = (top2[:, 1] - top2[:, 0]) > 2.5 * dl
        n_clear += clear.sum()
        assert (probs[b].argmax(-1) == l_ref.argmax(-1))[clear].all()
        rc, rl, rs = vr.greedy_decode(p_ref[None])
        if clear[1:rl[0] + 2].all():
            assert lengths[b] == rl[0] and np.array_equal(chars[b], rc[0])
            assert texts[b] == "".join(m.label(int(i)) for i in rc[0][:rl[0]])
            tol = float((0.55 * dl[1:rl[0] + 1] + 1e-6).sum())
            assert abs(scores[b] - rs[0]) <= tol, (scores[b], rs[0], tol)
    assert n_clear > 0.9 * len(imgs) * 25
    rm.close()
    m.close()


def test_batches_are_bit_identical_and_stable():
    """Batch sizes from 1 past the eager / graph switch (8192 tokens = 41 images of 197), mixed image sizes: the last image comes out
    bit-identical to the same image alone, three calls in a row (graph capture on the second, replay on the third)."""
    m = eng.vit_model_load(model_path("vitstr_tiny", "f16"), 0, 48, head_tokens=25)
    imgs = word_crops(48, seed=21)
    for B in (1, 2, 5, 13, 41, 42, 48):
        alone = recognize(m, imgs[B - 1:B])
        for rep in range(3):
            got = recognize(m, imgs[:B])
            assert all(np.array_equal(a[B - 1], w[0]) for a, w in zip(got, alone)), (B, rep)
    m.close()


def test_async_batches_interleave_with_classification():
    m = eng.vit_model_load(model_path("vitstr_tiny", "f16"), 0, 8, head_tokens=25)
    gray = gf.synthetic_gray_images(3, m.img_size, seed=9)
    cls_before = eng.vit_predict(m, gray, 5, want_logits=True)
    batches = [word_crops(8, seed=30), word_crops(5, seed=31)]
    want = [recognize(m, x, f32=False)[1:] for x in batches]
    L = eng.lib()
    for order in ((0, "cls", 1), (0, 1, "cls")):
        outs = {}
        for step in order:
            if step == "cls":
                got = eng.vit_predict(m, gray, 5, want_logits=True)
                assert all(np.array_equal(a, b) for a, b in zip(got, cls_before))
                continue
            x = [np.ascontiguousarray(a) for a in batches[step]]
            B = len(x)
            o = (np.empty((B, 24), np.int32), np.empty(B, np.int32), np.empty(B, np.float64), np.empty((B, 25, m.num_classes), np.float32))
            ptrs = (C.c_void_p * B)(*[a.ctypes.data for a in x])
            nx = (C.c_int * B)(*[a.shape[1] for a in x])
            ny = (C.c_int * B)(*[a.shape[0] for a in x])
            assert L.vitb200_recognize_u8_async(m.handle, ptrs, nx, ny, B, *[a.ctypes.data for a in o]) == 0
            outs[step] = o
        assert L.vitb200_sync(m.handle) == 0
        for i in (0, 1):
            assert all(np.array_equal(a, b) for a, b in zip(outs[i], want[i])), (order, i)
    got = eng.vit_predict(m, gray, 5, want_logits=True)
    assert all(np.array_equal(a, b) for a, b in zip(got, cls_before))
    m.close()


def test_launch_count():
    for cfg in ("vitstr_micro", "vitstr_tiny"):
        m = eng.vit_model_load(model_path(cfg, "f16"), 0, 4, head_tokens=25)
        L = m.hparams.num_hidden_layers
        for rep in range(3):  # eager, capture, replay
            eng.vitstr_recognize_u8(m, word_crops(3, seed=4))
            assert m.last_launch_count() == 3 + 7 * L + 4, (cfg, rep, m.last_launch_count())
        eng.vitstr_preprocess_u8(m, word_crops(3, seed=4))
        assert m.last_launch_count() == 1
        m.close()


def test_rejections_leave_the_engine_intact():
    path = model_path("vitstr_tiny", "f16")
    m = eng.vit_model_load(path, 0, 2, head_tokens=25)
    imgs = word_crops(2, seed=40)
    want = recognize(m, imgs)
    cases = [([np.zeros((1, 40, 3), np.uint8)], "2x2"), ([np.zeros((40, 1, 3), np.uint8)], "2x2"), ([], "batch"), (word_crops(3, seed=1), "batch")]
    for bad, what in cases:
        with pytest.raises(eng.VitB200Error) as ei:
            recognize(m, bad)
        assert what in str(ei.value)
        assert all(np.array_equal(a, b) for a, b in zip(recognize(m, imgs), want)), what
    m.close()

    rgb = eng.vit_model_load(model_path("micro", "f16"), 0, 2)
    x = gf.synthetic_images(2, rgb.img_size, seed=3)
    before = eng.vit_predict(rgb, x, 5, want_logits=True)
    with pytest.raises(eng.VitB200Error) as ei:
        eng.vitstr_recognize_u8(rgb, imgs)
    assert "grayscale" in str(ei.value) and "3-channel" in str(ei.value)
    assert all(np.array_equal(a, b) for a, b in zip(eng.vit_predict(rgb, x, 5, want_logits=True), before))
    rgb.close()
    one = eng.vit_model_load(path, 0, 2, head_tokens=1)
    gray = gf.synthetic_gray_images(2, one.img_size, seed=3)
    before = eng.vit_predict(one, gray, 5, want_logits=True)
    with pytest.raises(eng.VitB200Error) as ei:
        eng.vitstr_recognize_u8(one, imgs)
    assert "head_tokens" in str(ei.value)
    assert all(np.array_equal(a, b) for a, b in zip(eng.vit_predict(one, gray, 5, want_logits=True), before))
    one.close()
    m = eng.vit_model_load(path, 0, 2, head_tokens=25)
    assert all(np.array_equal(a, b) for a, b in zip(recognize(m, imgs), want))
    m.close()
