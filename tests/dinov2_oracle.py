"""Hugging Face DINOv2 as an independent float64 oracle for LayerScale, register tokens, the class-plus-patch-mean classifier and SwiGLU
MLPs (vitb200_arch), for tests.

The four HF classes (Dinov2Model, Dinov2ForImageClassification, Dinov2WithRegistersModel, Dinov2WithRegistersForImageClassification)
are built from a config under torch.manual_seed.  Matrix weights (linear layers, patch kernel, classifier) are rounded to f16, as the
engine stores them; LayerNorms are kept away from the identity; every LayerScale gamma is drawn log-uniformly over [1e-5, 1], so that a
dropped or misapplied gamma shows.  With swiglu (use_swiglu_ffn, ViT-g's Dinov2SwiGLUFFN) every block's MLP is weights_in [2 F][D] and
weights_out [D][F], F = (int(4 D * 2 / 3) + 7) // 8 * 8 (344 for D = 128, 4096 for ViT-g's D = 1536).  The model is saved as model.safetensors + config.json and converted with vit.cpp_b200/convert.py
(with --img-size when the geometry asks for it); the oracle runs the same weights in float64 at the converted input size, where HF
resamples its position embeddings at run time."""
import numpy as np

from tests.hf_oracle import init_model

# name: (hidden, heads, layers, patch, config image size, register tokens, converted image size or None)
GEOMETRIES = {
    "micro": (128, 2, 2, 14, 70, 0, 56),         # config grid 5 x 5, converted to 4 x 4: 17 tokens (the resampling runs)
    "micro_reg": (128, 2, 2, 14, 70, 4, 56),     # the same with 4 registers: 21 tokens
    "s14_reg4": (384, 6, 2, 14, 196, 4, None),   # S/14 with 4 registers at 196: 201 tokens (split-precision wgmma attention)
    "b14_reg4": (768, 12, 2, 14, 518, 4, 224),   # B/14 with 4 registers from a 518 config at 224: 261 tokens (mma.sync attention)
    "l14": (1024, 16, 2, 14, 224, 0, None),      # L/14 at 224: 257 tokens
    "g14_reg4": (1536, 24, 2, 14, 518, 4, 224),  # the ViT-g/14 block (F = 4096 with swiglu) with 4 registers from a 518 config at 224
}
NUM_LABELS = 10


def build_hf(geometry: str, classifier: bool = True, seed: int = 0, swiglu: bool = False):
    """The float32 HF model (matrix weights f16-valued) of a geometry: a registers geometry builds the WithRegisters classes; swiglu:
    use_swiglu_ffn."""
    import transformers as tr
    D, H, L, P, S, R, _ = GEOMETRIES[geometry]
    kw = dict(hidden_size=D, num_attention_heads=H, num_hidden_layers=L, patch_size=P, image_size=S, mlp_ratio=4, hidden_act="gelu",
              layer_norm_eps=1e-6, num_labels=NUM_LABELS, use_swiglu_ffn=swiglu)
    if R:
        cfg = tr.Dinov2WithRegistersConfig(num_register_tokens=R, **kw)
        cls = tr.Dinov2WithRegistersForImageClassification if classifier else tr.Dinov2WithRegistersModel
    else:
        cfg = tr.Dinov2Config(**kw)
        cls = tr.Dinov2ForImageClassification if classifier else tr.Dinov2Model
    # the mask token is [1][D]: drawn as a matrix, though the engine never reads it
    return init_model(cls, cfg, seed, norms=("norm",), f32=("position_embeddings", "register_tokens", "cls_token"))


def convert_size(geometry: str):
    """The --img-size the geometry converts with, or None for the config's image size."""
    return GEOMETRIES[geometry][6]


def image_size(geometry: str) -> int:
    """The input size of the converted model."""
    return convert_size(geometry) or GEOMETRIES[geometry][4]


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
