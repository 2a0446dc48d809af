"""What the Hugging Face oracles of tests/clip_oracle.py, dinov2_oracle.py and siglip_oracle.py share: a model built from a config under
torch.manual_seed with its weights redrawn, and its conversion to GGUF with vit.cpp_b200/convert.py."""
import os

import numpy as np

from tests.util import pkg


def init_model(cls, cfg, seed: int, norms, f32):
    """cls(cfg), float32 in eval mode, built under torch.manual_seed(seed), then every parameter redrawn in named_parameters order so
    that attention and the MLP activation are far from linear:

        LayerScale lambda1 (DINOv2)       log-uniform over [1e-5, 1], so that a dropped or misapplied gamma shows
        a name containing one of `norms`  1 + 0.2 randn (weight), 0.2 randn (bias): LayerNorms away from the identity
        any other bias                    0.05 randn
        a matrix (2 or more dimensions)   randn / sqrt(fan in), rounded to f16 as the engine stores it, unless its name contains one of
                                          `f32` (the embeddings the engine keeps in f32)
        anything else                     0.5 randn: class token, registers, positions, probe"""
    import torch
    torch.manual_seed(seed)
    m = cls(cfg).float().eval()
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "lambda1" in name:
                p.copy_(torch.exp(torch.empty_like(p).uniform_(np.log(1e-5), 0.0)))
            elif any(s in name for s in norms):
                p.copy_((1.0 if name.endswith("weight") else 0.0) + 0.2 * torch.randn_like(p))
            elif name.endswith("bias"):
                p.copy_(0.05 * torch.randn_like(p))
            elif p.ndim >= 2 and not any(s in name for s in f32):
                p.copy_((torch.randn_like(p) / p[0].numel() ** 0.5).half().float())
            else:
                p.copy_(0.5 * torch.randn_like(p))
    return m


def save_and_convert(model, directory: str, name: str, img_size=None) -> str:
    """save_pretrained + convert.py (the CLI's code path, with --img-size when img_size is given) -> the GGUF path, directory/name.gguf."""
    model.save_pretrained(directory)
    out = os.path.join(directory, f"{name}.gguf")
    pkg.convert.main([os.path.join(directory, "model.safetensors"), out, "--hf-config", os.path.join(directory, "config.json")] +
                     (["--img-size", str(img_size)] if img_size else []))
    return out
