"""Generate the head-dim-80 fixtures tests/golden/h80_*.npz from the UNMODIFIED reference (oracle/_ref/libvitref.so, built by
`make -C oracle ref`).  Run in the dev container:  python tests/golden/make_golden_head80.py

The models are synthetic legacy-ggml files (vit.cpp_b200/ggml_file.py write_synthetic) with hidden 160 and 2 heads, so every attention
head is 80 columns wide, as in ViT-H/14.  Each fixture holds the reference's pre-softmax logits and probabilities (vit_predict,
reference vit.cpp:1004-1075) for 8 seeded synthetic images, plus the sha256 of the model file so a drifting numpy RNG is detected."""
import hashlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests.util import gf  # noqa: E402
from oracle import ref  # noqa: E402

# name: (hidden, layers, heads, patch, img)
CASES = {
    "h80_micro": (160, 2, 2, 16, 64),    # 17 tokens: the split-precision form of the kernel
    "h80_h14": (160, 2, 2, 14, 224),     # 257 tokens, ViT-H/14's at 224 px: the f16-operand form
}
N_IMAGES, IMAGE_SEED = 8, 1234


def write_model(path: str, name: str) -> None:
    gf.write_synthetic(path, CASES[name], 1)


def sha256(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def main():
    out_dir = os.path.dirname(os.path.abspath(__file__))
    with tempfile.TemporaryDirectory() as tmp:
        for name in CASES:
            path = os.path.join(tmp, f"{name}.bin")
            write_model(path, name)
            m = ref.RefModel(path)
            imgs = gf.synthetic_images(N_IMAGES, m.img, seed=IMAGE_SEED)
            probs, logits = m.predict_batch(imgs, n_threads=8)
            np.savez_compressed(os.path.join(out_dir, f"{name}_f16.npz"), logits=logits, probs=probs, image_seed=IMAGE_SEED,
                                n_images=N_IMAGES, model_sha256=sha256(path))
            print(name, "top1", logits.argmax(1), "sha", sha256(path)[:12])
            m.close()


if __name__ == "__main__":
    main()
