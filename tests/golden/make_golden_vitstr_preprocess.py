"""Generate tests/golden/vitstr_preprocess.npz: u8 RGB images and what the ViTSTR extension's own vit_image_preprocess
(reference extensions/vitstr.cpp:135-201, compiled into oracle/_ref/libvitstrref.so) makes of them at the vitstr_micro geometry
(img_size 96), so that the bit-exact check of the GPU preprocess also runs where the compiled extension is absent.
Run in the dev container:  python tests/golden/make_golden_vitstr_preprocess.py

The images are stored back to back in `pixels` (uint8), with `shapes` [n][3] = (height, width, 3); `images_f32` is [n][96][96]."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import vitstr_reference as vr  # noqa: E402

S = 96
SIZES = [(2, 2), (5, 17), (97, 3), (32, 120), (S, S), (40, 23)]  # (height, width), random colour pixels


def images():
    rng = np.random.default_rng(2024)
    out = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in SIZES]
    out.append(np.zeros((7, 30, 3), np.uint8))
    out.append(np.full((30, 7, 3), 255, np.uint8))
    return out


def main():
    imgs = images()
    f32 = np.stack([vr.preprocess(im, S) for im in imgs])
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "vitstr_preprocess.npz")
    np.savez_compressed(dst, pixels=np.concatenate([im.reshape(-1) for im in imgs]), shapes=np.array([im.shape for im in imgs], np.int32),
                        images_f32=f32, img_size=S)
    print(dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
