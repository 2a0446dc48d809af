"""Hugging Face image processors on the GPU (vitb200_set_image_proc): the pixels of the u8 entry points against the PIL backends of
transformers' CLIP, SigLIP and Bit (DINOv2) processors, bit for bit, on a mixed batch per configuration; batch independence and
back-to-back asynchronous calls; CLIP, SigLIP and DINOv2 towers end to end against the f32 entry points on the processor's
pixel_values; and the interface's refusals."""

import numpy as np
import pytest

from tests.util import pkg, gf, model_path

eng = pkg.engine
pytestmark = pytest.mark.gpu
IMAGENET_MEAN, IMAGENET_STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def _processors():
    """name -> (PIL-backend processor, the model's img_size)."""
    import transformers as tr
    return {
        "clip224": (tr.CLIPImageProcessorPil(), 224),
        "clip336": (tr.CLIPImageProcessorPil(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336}), 336),
        "siglip224": (tr.SiglipImageProcessorPil(), 224),
        "siglip384": (tr.SiglipImageProcessorPil(size={"height": 384, "width": 384}), 384),
        "dinov2": (tr.BitImageProcessorPil(size={"shortest_edge": 256}, crop_size={"height": 224, "width": 224}, image_mean=IMAGENET_MEAN,
                                           image_std=IMAGENET_STD), 224),
        "bilinear224": (tr.SiglipImageProcessorPil(resample=2), 224),
    }


def _images(S, seed=0):
    """One mixed batch: heavy downscaling, upscaling, an image at the target size (both passes skipped in the exact-size configurations),
    one axis at the target size, odd crop margins, 1 x N and N x 1, random, saturated and checkerboard content."""
    rng = np.random.default_rng(seed)
    rand = lambda h, w: rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    checker = ((np.indices((61, 97)).sum(0) % 2) * 255).astype(np.uint8)[..., None].repeat(3, 2)
    sat = np.where(rng.random((150, 113, 1)) < 0.5, 0, 255).astype(np.uint8).repeat(3, 2)
    sat[:, :, 1] = 255 - sat[:, :, 1]
    return [rand(2000, 3000), rand(23, 17), rand(S, S), rand(S + 276, S), rand(403, 301), rand(1, 300), rand(300, 1), checker, sat,
            rand(S + 1, 2 * S + 3)]


def _hf_pixels(proc, imgs):
    """pixel_values of the PIL backend, CHW -> the engine's HWC."""
    from PIL import Image
    pv = proc([Image.fromarray(a) for a in imgs], return_tensors="np")["pixel_values"]
    return np.ascontiguousarray(np.asarray(pv, np.float32).transpose(0, 2, 3, 1))


def _rgb_model(S, max_batch=16):
    """A 1-layer RGB model of input size S, cached like tests.util.model_path's files."""
    import os
    from tests.util import CACHE
    os.makedirs(CACHE, exist_ok=True)
    path = os.path.join(CACHE, f"image-proc-{S}.bin")
    if not os.path.exists(path):
        gf.write_synthetic(path + f".tmp{os.getpid()}", (64, 1, 1, 16, S), 1, classes=10)
        os.replace(path + f".tmp{os.getpid()}", path)
    return eng.vit_model_load(path, 0, max_batch)


def _pixels(model, imgs):
    return eng.vit_image_preprocess_predict(model, imgs, predict=False)[0]


@pytest.mark.parametrize("name", ["clip224", "clip336", "siglip224", "siglip384", "dinov2", "bilinear224"])
def test_pixels_bit_for_bit(name):
    """images_f32_out of vitb200_forward_u8 == the processor's pixel_values, for the whole mixed batch and for each image alone."""
    proc, S = _processors()[name]
    m = _rgb_model(S)
    m.set_image_proc(proc.to_dict())
    imgs = _images(S)
    ref = _hf_pixels(proc, imgs)
    got = _pixels(m, imgs)
    assert m.last_launch_count() == 2
    bad = [i for i in range(len(imgs)) if not np.array_equal(got[i], ref[i])]
    assert not bad, [(imgs[i].shape, int((got[i] != ref[i]).sum()), float(np.abs(got[i] - ref[i]).max())) for i in bad]
    for i, a in enumerate(imgs):
        assert np.array_equal(_pixels(m, [a])[0], got[i]), i
    m.close()


def test_back_to_back_async_calls():
    """Two vitb200_forward_u8_async calls with different image sizes in flight at once (both pipeline slots, scratch sized per call):
    the logits of each equal vit_predict's on the processor's pixel_values."""
    proc, S = _processors()["clip224"]
    m = _rgb_model(S)
    m.set_image_proc(proc.to_dict())
    rng = np.random.default_rng(4)
    batches = [[rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shape]
               for shape in ([(900, 1300), (240, 230), (31, 500)], [(224, 224), (600, 2), (700, 650), (1200, 1100)])]
    outs, keep = [], []
    for imgs in batches:
        arrs, B, ptrs, nx, ny = eng._u8_batch(imgs)
        logits = np.empty((B, m.num_classes), np.float32)
        keep.append((arrs, ptrs, nx, ny))
        rc = eng.lib().vitb200_forward_u8_async(m.handle, ptrs, nx, ny, B, 0, None, logits.ctypes.data, None, None, 0)
        assert rc == 0, eng.lib().vitb200_last_error()
        outs.append(logits)
    assert eng.lib().vitb200_sync(m.handle) == 0
    for imgs, logits in zip(batches, outs):
        ref = eng.vit_predict(m, _hf_pixels(proc, imgs), topk=1, want_logits=True)[3]
        assert np.array_equal(logits, ref)
    m.close()


def _tower(kind, tmp_path, fp8=False):
    """A CLIP, SigLIP or DINOv2 micro tower converted with --hf-preprocessor, and its processor."""
    import json
    import os
    import transformers as tr
    from tests import clip_oracle, siglip_oracle, dinov2_oracle
    d = str(tmp_path / kind)
    if kind == "clip":
        model, S = clip_oracle.build_hf("micro"), 64
        proc = tr.CLIPImageProcessorPil(size={"shortest_edge": S}, crop_size={"height": S, "width": S})
    elif kind == "siglip":
        model, S = siglip_oracle.build_hf("micro"), 64
        proc = tr.SiglipImageProcessorPil(size={"height": S, "width": S})
    else:
        model, S = dinov2_oracle.build_hf("micro"), dinov2_oracle.image_size("micro")
        proc = tr.BitImageProcessorPil(size={"shortest_edge": 64}, crop_size={"height": S, "width": S}, image_mean=IMAGENET_MEAN,
                                       image_std=IMAGENET_STD)
    model.save_pretrained(d)
    pp = os.path.join(d, "preprocessor_config.json")
    with open(pp, "w") as f:
        json.dump(proc.to_dict(), f, default=int)
    out = os.path.join(d, f"{kind}.gguf")
    args = [os.path.join(d, "model.safetensors"), out, "--hf-config", os.path.join(d, "config.json"), "--hf-preprocessor", pp]
    pkg.convert.main(args + (["--img-size", str(S)] if kind == "dinov2" else []))
    return eng.vit_model_load(out, 0, 16, fp8=fp8), proc


@pytest.mark.parametrize("kind", ["clip", "siglip", "dinov2"])
def test_towers_end_to_end(kind, tmp_path):
    """A file converted with --hf-preprocessor loads with the processor set; vit_features_u8 and vit_image_preprocess_predict through it
    equal the f32 entry points on the processor's pixel_values, bit for bit; the FP8 engine once."""
    for fp8 in ((False, True) if kind == "siglip" else (False,)):
        m, proc = _tower(kind, tmp_path / str(fp8), fp8)
        assert m.image_proc == eng.image_proc_from_config(proc.to_dict(), m.img_size) | {
            "mean": [float(np.float32(x)) for x in proc.image_mean], "std": [float(np.float32(x)) for x in proc.image_std]}
        imgs = _images(m.img_size, seed=7)[1:]  # all but the 3000 x 2000 photo: the towers are 64 px
        pv = _hf_pixels(proc, imgs)
        tok_u8, pre_u8 = eng.vit_features_u8(m, imgs, prelogits=True)
        tok, pre = eng.vit_features(m, pv, prelogits=True)
        assert np.array_equal(tok_u8, tok) and np.array_equal(pre_u8, pre)
        f32, probs, idx, val, logits = eng.vit_image_preprocess_predict(m, imgs)
        assert np.array_equal(f32, pv)
        p_ref, i_ref, v_ref, l_ref = eng.vit_predict(m, pv, want_logits=True)
        assert np.array_equal(logits, l_ref) and np.array_equal(probs, p_ref) and np.array_equal(idx, i_ref)
        m.close()


def test_interface():
    """bilinear = 1 is refused with a processor; set_image_proc(None) restores vit.cpp's preprocessing bit for bit; a ViTSTR engine
    refuses a processor; the getter returns what was set, and all zero (None) after clearing it."""
    proc, S = _processors()["siglip224"]
    imgs = _images(S, seed=2)[1:5]
    m, plain = _rgb_model(S), _rgb_model(S)
    assert m.image_proc is None
    before = _pixels(plain, imgs)
    m.set_image_proc(proc.to_dict())
    assert m.image_proc["height"] == 224 and m.image_proc["resample"] == 3
    with pytest.raises(eng.VitB200Error, match="bilinear = 1: the engine's image processor fixes the resample"):
        eng.vit_image_preprocess_predict(m, imgs, bilinear=True, predict=False)
    with pytest.raises(eng.VitB200Error, match="bilinear = 1"):
        eng.vit_features_u8(m, imgs, bilinear=True)
    m.set_image_proc(None)
    assert m.image_proc is None
    assert np.array_equal(_pixels(m, imgs), before)
    assert m.last_launch_count() == 1
    with pytest.raises(eng.VitB200Error, match="image_proc.resample = 1"):
        m.set_image_proc(dict(eng.image_proc_from_config(proc.to_dict(), S), resample=1))
    assert m.image_proc is None  # a refused processor changes nothing
    vs = eng.vit_model_load(model_path("vitstr_micro", "f16"), 0, 2, head_tokens=25)
    with pytest.raises(eng.VitB200Error, match="image_proc: this model takes 1-channel input"):
        vs.set_image_proc(dict(proc.to_dict(), size={"height": 96, "width": 96}))
    for x in (m, plain, vs):
        x.close()
