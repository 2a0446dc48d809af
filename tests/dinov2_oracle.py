"""Hugging Face DINOv2 as an independent float64 oracle for LayerScale, register tokens and the class-plus-patch-mean classifier
(vitb200_arch), for tests.

The four HF classes (Dinov2Model, Dinov2ForImageClassification, Dinov2WithRegistersModel, Dinov2WithRegistersForImageClassification)
are built from a config under torch.manual_seed.  Matrix weights (linear layers, patch kernel, classifier) are rounded to f16, as the
engine stores them; LayerNorms are kept away from the identity; every LayerScale gamma is drawn log-uniformly over [1e-5, 1], so that a
dropped or misapplied gamma shows.  The model is saved as model.safetensors + config.json and converted with vit.cpp_b200/convert.py
(with --img-size when the geometry asks for it); the oracle runs the same weights in float64 at the converted input size, where HF
resamples its position embeddings at run time."""
import os

import numpy as np

from tests.util import pkg

# name: (hidden, heads, layers, patch, config image size, register tokens, converted image size or None)
GEOMETRIES = {
    "micro": (128, 2, 2, 14, 70, 0, 56),         # config grid 5 x 5, converted to 4 x 4: 17 tokens (the resampling runs)
    "micro_reg": (128, 2, 2, 14, 70, 4, 56),     # the same with 4 registers: 21 tokens
    "s14_reg4": (384, 6, 2, 14, 196, 4, None),   # S/14 with 4 registers at 196: 201 tokens (split-precision wgmma attention)
    "b14_reg4": (768, 12, 2, 14, 518, 4, 224),   # B/14 with 4 registers from a 518 config at 224: 261 tokens (mma.sync attention)
    "l14": (1024, 16, 2, 14, 224, 0, None),      # L/14 at 224: 257 tokens
}
NUM_LABELS = 10


def build_hf(geometry: str, classifier: bool = True, seed: int = 0):
    """The float32 HF model (matrix weights f16-valued) of a geometry: a registers geometry builds the WithRegisters classes."""
    import torch
    import transformers as tr
    D, H, L, P, S, R, _ = GEOMETRIES[geometry]
    kw = dict(hidden_size=D, num_attention_heads=H, num_hidden_layers=L, patch_size=P, image_size=S, mlp_ratio=4, hidden_act="gelu",
              layer_norm_eps=1e-6, num_labels=NUM_LABELS)
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
    out = os.path.join(directory, "dinov2.gguf")
    conv = GEOMETRIES[geometry][6]
    pkg.convert.main([os.path.join(directory, "model.safetensors"), out, "--hf-config", os.path.join(directory, "config.json")] +
                     (["--img-size", str(conv)] if conv else []))
    return out


def backbone(model):
    """The encoder of any of the four classes."""
    for name in ("dinov2", "dinov2_with_registers"):
        if hasattr(model, name):
            return getattr(model, name)
    return model


def hf_outputs(model, imgs) -> dict:
    """float64 oracle on images float32 [B][S][S][3] (NHWC): `logits` (the classifier's, or pooler_output without one), `prelogits`
    (the head's input: [LN(cls) || mean LN(patches)] with a classifier, pooler_output without), hidden_states[i], i = 0 .. L."""
    import torch
    m = model.double()
    x = torch.from_numpy(np.ascontiguousarray(np.asarray(imgs, np.float64).transpose(0, 3, 1, 2)))
    R = getattr(m.config, "num_register_tokens", 0)
    with torch.no_grad():
        o = backbone(m)(pixel_values=x, output_hidden_states=True)
        seq = o.last_hidden_state
        if hasattr(m, "classifier"):
            pre = torch.cat([seq[:, 0], seq[:, 1 + R:].mean(dim=1)], dim=1)
            logits = m.classifier(pre)
        else:
            pre = logits = o.pooler_output
    model.float()
    return {"logits": logits.numpy(), "prelogits": pre.numpy(), "hidden_states": [h.numpy() for h in o.hidden_states]}
