"""Hugging Face DINOv2 with SwiGLU MLPs (use_swiglu_ffn, ViT-g's Dinov2SwiGLUFFN) as an independent float64 oracle for
vitb200_arch.activation = 4, for tests.

The models are built as tests/dinov2_oracle.py builds them -- the four classes from a config under torch.manual_seed, f16-valued matrix
weights, LayerNorms away from the identity, gamma log-uniform over [1e-5, 1] -- with use_swiglu_ffn set, so every block's MLP is
weights_in [2 F][D] and weights_out [D][F], F = (int(4 D * 2 / 3) + 7) // 8 * 8 (344 for D = 128, 4096 for ViT-g's D = 1536).
hf_outputs and backbone are tests/dinov2_oracle.py's."""
import os

import numpy as np

from tests.util import pkg
from tests.dinov2_oracle import GEOMETRIES as _DINOV2, NUM_LABELS, backbone, hf_outputs  # noqa: F401 (re-exported)

# name: (hidden, heads, layers, patch, config image size, register tokens, converted image size or None): DINOv2's geometries and the
# ViT-g/14 block (F = 4096) with 4 registers from a 518 config at 224, 261 tokens
GEOMETRIES = dict(_DINOV2, g14_reg4=(1536, 24, 2, 14, 518, 4, 224))


def build_hf(geometry: str, classifier: bool = True, seed: int = 0):
    """The float32 HF SwiGLU model (matrix weights f16-valued) of a geometry: a registers geometry builds the WithRegisters classes."""
    import torch
    import transformers as tr
    D, H, L, P, S, R, _ = GEOMETRIES[geometry]
    kw = dict(hidden_size=D, num_attention_heads=H, num_hidden_layers=L, patch_size=P, image_size=S, mlp_ratio=4, hidden_act="gelu",
              layer_norm_eps=1e-6, num_labels=NUM_LABELS, use_swiglu_ffn=True)
    if R:
        cfg = tr.Dinov2WithRegistersConfig(num_register_tokens=R, **kw)
        cls = tr.Dinov2WithRegistersForImageClassification if classifier else tr.Dinov2WithRegistersModel
    else:
        cfg = tr.Dinov2Config(**kw)
        cls = tr.Dinov2ForImageClassification if classifier else tr.Dinov2Model
    torch.manual_seed(seed)
    m = cls(cfg).float().eval()
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "lambda1" in name:
                p.copy_(torch.exp(torch.empty_like(p).uniform_(np.log(1e-5), 0.0)))   # log-uniform over [1e-5, 1]
            elif "norm" in name:
                p.copy_((1.0 if name.endswith("weight") else 0.0) + 0.2 * torch.randn_like(p))
            elif name.endswith("bias"):
                p.copy_(0.05 * torch.randn_like(p))
            elif p.ndim >= 2 and "position_embeddings" not in name and "register_tokens" not in name and "cls_token" not in name:
                fan_in = p[0].numel()
                p.copy_((torch.randn_like(p) / fan_in ** 0.5).half().float())   # f16-valued, as the engine stores them
            else:
                p.copy_(0.5 * torch.randn_like(p))                               # cls, registers, positions, mask token (f32)
    return m


def image_size(geometry: str) -> int:
    """The input size of the converted model."""
    _, _, _, _, S, _, conv = GEOMETRIES[geometry]
    return conv or S


def save_and_convert(model, directory: str, geometry: str) -> str:
    """save_pretrained + convert.py (the CLI's code path, --img-size when the geometry converts to another size) -> the GGUF path."""
    model.save_pretrained(directory)
    out = os.path.join(directory, "dinov2_swiglu.gguf")
    conv = GEOMETRIES[geometry][6]
    pkg.convert.main([os.path.join(directory, "model.safetensors"), out, "--hf-config", os.path.join(directory, "config.json")] +
                     (["--img-size", str(conv)] if conv else []))
    return out
