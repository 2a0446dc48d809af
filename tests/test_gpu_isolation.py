"""Every image is an independent unit, non-finite values included: an image holding NaN, or pixels that overflow f16 (patchify rounds
them to Inf), must not change a single bit of its batch mates' outputs, nor of any later call's.  "Clean" below is what the same
images give on a fresh engine, which batch invariance makes bit-exact.

Geometries: micro (17 tokens) and tiny (197) run the wgmma attention, whose 224-row key box spans 13 micro images; large384x2 (577)
the 16-warp and p8 (785) the 8-warp mma.sync kernel; h80_micro (17) and h80_h14 (257), with 80-column heads, the split-precision and
the f16 form of the head-dim-80 kernel; a CLIP micro tower (pre-norm) and a DINOv2 micro model with registers and the
class-plus-patch-mean pool; and a ViTSTR model through the text recognition entry point."""
import numpy as np
import pytest

from tests import clip_oracle as co
from tests import dinov2_oracle as do
from tests.hf_oracle import save_and_convert
from tests.test_gpu_head80 import _model_path as head80_model_path, mg
from tests.util import pkg, gf, model_path

eng = pkg.engine
pytestmark = pytest.mark.gpu

GEOS = ["micro", "tiny", "large384x2", "p8", "h80_micro", "h80_h14", "clip_micro", "dinov2_micro_reg"]
GRAPH_TOKENS = 8192   # calls of batch * N <= this many tokens run through a cached CUDA graph (captured on an argument set's 2nd call)
POISONS = ["nan_pixel", "f16_overflow"]
TOPK = 5

_paths = {}


def _path(geo, tmp_path_factory):
    if geo not in _paths:
        if geo == "clip_micro":
            d = str(tmp_path_factory.mktemp("clip_micro"))
            _paths[geo] = save_and_convert(co.build_hf("micro", "quick_gelu"), d, "clip")
        elif geo == "dinov2_micro_reg":
            d = str(tmp_path_factory.mktemp("dinov2_micro_reg"))
            _paths[geo] = save_and_convert(do.build_hf("micro_reg", True), d, "dinov2", do.convert_size("micro_reg"))
        elif geo in mg.CASES:
            _paths[geo] = head80_model_path(geo, tmp_path_factory)
        else:
            _paths[geo] = model_path(geo, "f16")
    return _paths[geo]


def _poison(img, kind):
    """One NaN pixel in the last patch, or every pixel 1e6 (f16 Inf after patchify)."""
    img = img.copy()
    if kind == "nan_pixel":
        img[-1, -1, -1] = np.nan
    else:
        img[:] = 1e6
    return img


def _images(m, n, seed):
    return gf.synthetic_images(n, m.img_size, seed=seed)


def _predict(m, imgs):
    probs, idx, val, logits = eng.vit_predict(m, imgs, TOPK, want_logits=True)
    return {"probs": probs, "logits": logits, "topk_idx": idx, "topk_val": val}


def _features(m, imgs):
    tok, pre = eng.vit_features(m, imgs, layers=None, norm=True, tokens=True, prelogits=True)
    return {"tokens": tok, "prelogits": pre}


def _forward_async(m, imgs):
    B, nc = imgs.shape[0], m.num_classes
    o = {"probs": np.empty((B, nc), np.float32), "logits": np.empty((B, nc), np.float32), "topk_idx": np.empty((B, TOPK), np.int32),
         "topk_val": np.empty((B, TOPK), np.float32)}
    x = np.ascontiguousarray(imgs, np.float32)
    eng._check(eng.lib().vitb200_forward_async(m.handle, x.ctypes.data, B, o["probs"].ctypes.data, o["logits"].ctypes.data,
                                               o["topk_idx"].ctypes.data, o["topk_val"].ctypes.data, TOPK), "vitb200_forward_async")
    eng._check(eng.lib().vitb200_sync(m.handle), "vitb200_sync")
    return o


_dev_bufs = {}


def _forward_device(m, imgs):
    """vitb200_forward_device with the same device buffers on every call of a batch size, so its graph is captured and replayed."""
    import torch
    B, nc = imgs.shape[0], m.num_classes
    key = (m.handle.value, imgs.shape, nc)
    if key not in _dev_bufs:
        _dev_bufs[key] = {"img": torch.empty(imgs.shape, dtype=torch.float32, device="cuda"),
                          "probs": torch.empty((B, nc), dtype=torch.float32, device="cuda"),
                          "logits": torch.empty((B, nc), dtype=torch.float32, device="cuda"),
                          "topk_idx": torch.empty((B, TOPK), dtype=torch.int32, device="cuda"),
                          "topk_val": torch.empty((B, TOPK), dtype=torch.float32, device="cuda")}
    d = _dev_bufs[key]
    d["img"].copy_(torch.from_numpy(np.ascontiguousarray(imgs, np.float32)))
    torch.cuda.synchronize()
    eng._check(eng.lib().vitb200_forward_device(m.handle, d["img"].data_ptr(), B, d["probs"].data_ptr(), d["logits"].data_ptr(),
                                                d["topk_idx"].data_ptr(), d["topk_val"].data_ptr(), TOPK, None), "vitb200_forward_device")
    eng._check(eng.lib().vitb200_sync(m.handle), "vitb200_sync")
    return {k: d[k].cpu().numpy() for k in ("probs", "logits", "topk_idx", "topk_val")}


ENTRIES = {"forward": _predict, "forward_async": _forward_async, "forward_device": _forward_device, "features": _features}


def _same(got, want, rows, what):
    for k in want:
        assert np.array_equal(got[k][rows], want[k][rows]), (what, k)


def _check_poisoned_rows(out, rows, C):
    for r in rows:
        assert not np.isfinite(out["logits"][r]).all(), r
        idx = out["topk_idx"][r]
        assert ((idx == -1) | ((idx >= 0) & (idx < C))).all(), (r, idx.tolist())


def _batch(geo):
    """16 images of the 17-token geometries (13 of them span the wgmma kernel's 224-row box), or five for the larger token counts."""
    return {"micro": 16, "h80_micro": 16, "clip_micro": 16, "dinov2_micro_reg": 16}.get(geo, 5)


@pytest.mark.parametrize("kind", POISONS)
@pytest.mark.parametrize("geo", GEOS)
def test_batch_mates_are_untouched(geo, kind, tmp_path_factory):
    """Poisoned first, middle and last images: every other image's logits, probabilities, top-k and features (tokens after the last
    block, prelogits) are bit-identical to its clean result; the poisoned images' logits are not all finite and their top-k ids are
    -1 or in [0, C)."""
    path = _path(geo, tmp_path_factory)
    n = _batch(geo)
    fresh = eng.vit_model_load(path, 0, n)
    imgs = _images(fresh, n, seed=17)
    want = {**_predict(fresh, imgs), **_features(fresh, imgs)}
    fresh.close()
    bad = [0, n // 2, n - 1]
    x = imgs.copy()
    for b in bad:
        x[b] = _poison(x[b], kind)
    m = eng.vit_model_load(path, 0, n)
    got = {**_predict(m, x), **_features(m, x)}
    clean = [b for b in range(n) if b not in bad]
    _same(got, want, clean, "batch mates")
    _check_poisoned_rows(got, bad, m.num_classes)
    # and the engine is clean again for the next call
    after = _predict(m, imgs)
    _same(after, {k: want[k] for k in after}, slice(None), "after")
    m.close()


def _stale_sizes(m):
    """(small, large): a batch that replays a graph, and the smallest that launches eagerly."""
    return 5, GRAPH_TOKENS // m.n_tokens + 1


@pytest.mark.parametrize("kind", POISONS)
@pytest.mark.parametrize("geo", GEOS)
def test_stale_rows_of_an_earlier_call_are_never_read(geo, kind, tmp_path_factory):
    """A full max_batch call holds poisoned images in the slots right after the next calls' batches; then clean calls with smaller
    batches, through every entry point (vitb200_forward, _forward_async + _sync, _forward_device, vitb200_features), eagerly (a batch
    above the graph bound) and through graph capture and replay (a batch below it, six calls so that both pipeline slots capture and
    replay), must equal a fresh engine's results bit for bit."""
    path = _path(geo, tmp_path_factory)
    probe = eng.vit_model_load(path, 0, 1)
    small, large = _stale_sizes(probe)
    probe.close()
    mb = large + 2
    fresh = eng.vit_model_load(path, 0, mb)
    imgs = _images(fresh, mb, seed=23)
    want = {(name, B): fn(fresh, imgs[:B]) for name, fn in ENTRIES.items() for B in (small, large)}
    fresh.close()
    x = imgs.copy()
    for slot in (small, large):
        x[slot] = _poison(x[slot], kind)
    m = eng.vit_model_load(path, 0, mb)
    for name, fn in ENTRIES.items():
        for B, reps in ((small, 6), (large, 1)):
            _predict(m, x)    # the poisoned full batch, right before
            for rep in range(reps):
                _same(fn(m, imgs[:B]), want[(name, B)], slice(None), (name, B, rep))
    m.close()


def _recognize(m, imgs):
    texts, scores, chars, lengths = eng.vitstr_recognize_u8(m, imgs)
    return {"scores": scores, "chars": chars, "lengths": lengths}


@pytest.mark.parametrize("kind", POISONS)
def test_text_recognition_after_a_poisoned_call(kind):
    """ViTSTR: a clean vitstr_recognize_u8 after a poisoned f32 call returns the fresh engine's characters, lengths and scores."""
    path = model_path("vitstr_micro", "f16")
    mb = 8
    rng = np.random.default_rng(4)
    crops = [rng.integers(0, 256, size=(int(rng.integers(24, 97)), int(rng.integers(64, 257)), 3), dtype=np.uint8) for _ in range(3)]
    fresh = eng.vit_model_load(path, 0, mb, head_tokens=25)
    want = _recognize(fresh, crops)
    fresh.close()
    m = eng.vit_model_load(path, 0, mb, head_tokens=25)
    gray = gf.synthetic_gray_images(mb, m.img_size, seed=6)
    for slot in range(len(crops), mb):    # every slot the recognition call does not use
        if kind == "nan_pixel":
            gray[slot, -1, -1] = np.nan
        else:
            gray[slot] = 1e6
    probs, idx, _ = eng.vit_predict(m, gray, TOPK)
    assert ((idx == -1) | ((idx >= 0) & (idx < m.num_classes))).all()
    for rep in range(6):
        _same(_recognize(m, crops), want, slice(None), rep)
    m.close()
