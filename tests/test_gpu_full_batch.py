"""The CLIP, DINOv2, SigLIP and SwiGLU towers at production batch sizes, where every GEMM runs many tiles per CTA on both MMA
warpgroups, the pools and the attention-pooling head run one CTA per image (per image and head), and the head GEMMs have M = batch.

The towers' own tests hold 3 images to the Hugging Face oracle.  Here those 3 images sit at positions 0, 128 (or the middle) and the
last of a full batch of distinct images, and every output -- logits, prelogits and the normalised last-layer tokens -- must equal, bit
for bit, what the same engine gives the 3 images alone; every other image must equal its own run alone and in consecutive batches of 7,
which put the image boundaries at other places in the GEMM tiles.  A tile, row band or pool CTA that reads or writes another image's
rows at full batch breaks the equality at the first wrong element."""
import time

import numpy as np
import pytest

from tests.util import pkg, gf
from tests import clip_oracle as co
from tests import dinov2_oracle as do
from tests import siglip_oracle as so
from tests.hf_oracle import save_and_convert

eng = pkg.engine
pytestmark = pytest.mark.gpu

# (family, geometry, activation or classifier, batch)
CASES = [("clip", "b32", "quick_gelu", 256), ("clip", "b32", "gelu_erf", 256), ("clip", "l14_336", "quick_gelu", 64),
         ("dinov2", "b14_reg4", True, 256), ("siglip", "b16_224", False, 256), ("siglip", "b16_256", True, 256),
         ("swiglu", "g14_reg4", True, 64)]
# the FP8 engine on one geometry per family
FP8 = [("clip", "b32", "quick_gelu", 256), ("dinov2", "b14_reg4", True, 256), ("siglip", "b16_224", False, 256),
       ("swiglu", "g14_reg4", True, 64)]
_built = {}


def _model(family, geo, variant, tmp_path_factory):
    """The tower's HF model (the seed its own test uses) converted to GGUF, once per module."""
    key = (family, geo, variant)
    if key not in _built:
        t0 = time.perf_counter()
        d = str(tmp_path_factory.mktemp(f"full_{family}_{geo}_{variant}"))
        if family == "clip":
            path = save_and_convert(co.build_hf(geo, variant), d, "clip")
        elif family == "dinov2":
            path = save_and_convert(do.build_hf(geo, variant), d, "dinov2", do.convert_size(geo))
        elif family == "siglip":
            path = save_and_convert(so.build_hf(geo, variant), d, "siglip")
        else:
            path = save_and_convert(do.build_hf(geo, variant, swiglu=True), d, "dinov2", do.convert_size(geo))
        print(f"{family} {geo} {variant}: HF model built and converted in {time.perf_counter() - t0:.1f} s (CPU)")
        _built[key] = path
    return _built[key]


def _run(m, imgs):
    """logits, prelogits (norm = 1) and the last layer's tokens after the final LayerNorm."""
    logits = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    tok, pre = eng.vit_features(m, imgs, norm=True, prelogits=True)
    return {"logits": logits, "prelogits": pre, "tokens": tok}


def _assert_rows(got, full, rows, what):
    for k in full:
        bad = [r for i, r in enumerate(rows) if not np.array_equal(got[k][i], full[k][r])]
        assert not bad, f"{what}: {k} of images {bad[:8]} differ from the full batch"


def _full_batch(family, geo, variant, B, fp8, tmp_path_factory, ragged=False):
    path = _model(family, geo, variant, tmp_path_factory)
    m = eng.vit_model_load(path, 0, B, fp8=fp8)
    try:
        S = m.img_size
        case = gf.synthetic_images(3, S, seed=3)  # the images the tower's own test holds to the oracle
        imgs = gf.synthetic_images(B, S, seed=1000 + B)
        at = [0, min(128, B // 2), B - 1]
        imgs[at] = case
        t0 = time.perf_counter()
        full = _run(m, imgs)
        t_full = time.perf_counter() - t0
        assert all(np.isfinite(v).all() for v in full.values())
        _assert_rows(_run(m, case), full, at, "the 3 oracle images alone")
        t0 = time.perf_counter()
        for s in range(0, B, 7):
            rows = list(range(s, min(s + 7, B)))
            _assert_rows(_run(m, imgs[rows]), full, rows, f"batch of 7 from image {s}")
        for r in range(B):
            if r not in at:
                _assert_rows(_run(m, imgs[r:r + 1]), full, [r], "alone")
        if ragged:
            _assert_rows(_run(m, imgs[:B - 1]), full, list(range(B - 1)), f"batch of {B - 1}")
        print(f"{family} {geo} {variant} fp8={fp8}: batch {B} in {t_full:.2f} s, the smaller batches in {time.perf_counter() - t0:.1f} s "
              "(wall, host side included)")
    finally:
        m.close()


@pytest.mark.parametrize("family,geo,variant,B", CASES, ids=[f"{f}-{g}-{v}" for f, g, v, _ in CASES])
def test_full_batch_equals_small_batches(family, geo, variant, B, tmp_path_factory):
    """CLIP b32 with QuickGELU also runs the ragged batch B - 1."""
    _full_batch(family, geo, variant, B, False, tmp_path_factory, ragged=(family, geo, variant) == ("clip", "b32", "quick_gelu"))


@pytest.mark.parametrize("family,geo,variant,B", FP8, ids=[f"{f}-{g}-{v}" for f, g, v, _ in FP8])
def test_full_batch_equals_small_batches_fp8(family, geo, variant, B, tmp_path_factory):
    _full_batch(family, geo, variant, B, True, tmp_path_factory)
