"""Hugging Face CLIP vision towers as an independent float64 oracle for the CLIP architecture (vitb200_arch), for tests.

A CLIPVisionModelWithProjection is built from a config under torch.manual_seed, with weights scaled so that attention and the MLP
activation are far from linear, and LayerNorms away from the identity.  Its matrix weights (the linear layers, the patch kernel and the
projection: what the engine stores as f16) are rounded to f16, so the oracle and the engine start from the same weights.  It is saved
as model.safetensors + config.json and converted with vit.cpp_b200/convert.py; the oracle runs the same weights in float64."""
import json
import os

import numpy as np

from tests.hf_oracle import init_model

# name: (hidden, heads, layers, patch, image, projection dim)
GEOMETRIES = {
    "micro": (128, 2, 2, 16, 64, 96),         # 17 tokens
    "b32": (768, 12, 2, 32, 224, 512),        # ViT-B/32 at 224: 50 tokens
    "l14_336": (1024, 16, 2, 14, 336, 768),   # ViT-L/14-336 (LLaVA's tower) cut to 2 layers: 577 tokens
}
HF_ACT = {"quick_gelu": "quick_gelu", "gelu_erf": "gelu"}


def build_hf(geometry: str, activation: str = "quick_gelu", seed: int = 0):
    """The float32 HF model (matrix weights f16-valued) for a geometry of GEOMETRIES; activation 'quick_gelu' or 'gelu_erf'."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    D, H, L, P, S, proj = GEOMETRIES[geometry]
    cfg = CLIPVisionConfig(hidden_size=D, intermediate_size=4 * D, num_attention_heads=H, num_hidden_layers=L, patch_size=P, image_size=S,
                           projection_dim=proj, hidden_act=HF_ACT[activation], layer_norm_eps=1e-5)
    # post_layernorm matches neither norm name: its weight and bias keep the 0.5 and 0.05 randn draws the bounds were measured with
    return init_model(CLIPVisionModelWithProjection, cfg, seed, norms=("layer_norm", "layrnorm"), f32=("position_embedding",))


def hf_outputs(model, imgs) -> dict:
    """float64 oracle on images float32 [B][S][S][3] (NHWC, the engine's layout): image_embeds, pooler_output and hidden_states[i],
    i = 0 .. L, as numpy float64."""
    import torch
    m = model.double()
    x = torch.from_numpy(np.ascontiguousarray(np.asarray(imgs, np.float64).transpose(0, 3, 1, 2)))
    with torch.no_grad():
        vo = m.vision_model(pixel_values=x, output_hidden_states=True)
        emb = m.visual_projection(vo.pooler_output)
    model.float()
    return {"image_embeds": emb.numpy(), "pooler_output": vo.pooler_output.numpy(), "hidden_states": [h.numpy() for h in vo.hidden_states]}


def write_config(directory: str, **fields) -> str:
    """A config.json for converter tests that need no model."""
    path = os.path.join(directory, "config.json")
    with open(path, "w") as f:
        json.dump(fields, f)
    return path
