"""Hugging Face SigLIP as an independent float64 oracle for the patch-only token rows, the attention-pooling head and PyTorch's tanh GELU
(vitb200_arch pools 2 and 3, activation 3), for tests.

SiglipVisionModel and SiglipForImageClassification are built from a config under torch.manual_seed.  Matrix weights (linear layers,
the attention-pooling head's in_proj / out_proj, patch kernel, classifier) are rounded to f16, as the engine stores them; LayerNorms are
kept away from the identity.  The model is saved as model.safetensors + config.json and converted with vit.cpp_b200/convert.py; the
oracle runs the same weights in float64."""
import numpy as np

from tests.hf_oracle import init_model

# name: (hidden, heads, layers, patch, image size)
GEOMETRIES = {
    "micro": (128, 2, 2, 16, 64),          # 16 tokens
    "b16_224": (768, 12, 2, 16, 224),      # 196 tokens: the split-precision wgmma attention
    "b16_256": (768, 12, 2, 16, 256),      # 256 tokens: the 16-warp mma.sync attention
    "l16_384": (1024, 16, 2, 16, 384),     # 576 tokens
}
NUM_LABELS = 10


def vision_config(geometry: str):
    import transformers as tr
    D, H, L, P, S = GEOMETRIES[geometry]
    return tr.SiglipVisionConfig(hidden_size=D, intermediate_size=4 * D, num_attention_heads=H, num_hidden_layers=L, patch_size=P,
                                 image_size=S, hidden_act="gelu_pytorch_tanh", layer_norm_eps=1e-6, attn_implementation="eager")


def build_hf(geometry: str, classifier: bool = False, seed: int = 0):
    """The float32 HF model (matrix weights f16-valued): SiglipForImageClassification or SiglipVisionModel."""
    import transformers as tr
    vc = vision_config(geometry)
    if classifier:
        cfg = tr.SiglipConfig(vision_config=vc.to_dict(), text_config=dict(hidden_size=64, intermediate_size=128, num_hidden_layers=1,
                                                                           num_attention_heads=1), num_labels=NUM_LABELS)
        cfg._attn_implementation = "eager"
        cls = tr.SiglipForImageClassification
    else:
        cfg, cls = vc, tr.SiglipVisionModel
    return init_model(cls, cfg, seed, norms=("norm",), f32=("position_embedding", "probe"))


def image_size(geometry: str) -> int:
    return GEOMETRIES[geometry][4]


def hf_outputs(model, imgs) -> dict:
    """float64 oracle on images float32 [B][S][S][3] (NHWC): `logits` (the classifier's, or pooler_output without one), `prelogits`
    (the head's input: the mean of last_hidden_state with a classifier, pooler_output without), hidden_states[i], i = 0 .. L, and
    last_hidden_state (post_layernorm of hidden_states[L])."""
    import torch
    m = model.double()
    x = torch.from_numpy(np.ascontiguousarray(np.asarray(imgs, np.float64).transpose(0, 3, 1, 2)))
    vt = m.vision_model
    with torch.no_grad():
        # SiglipVisionTransformer's own forward, step by step (the classifier class does not return the hidden states)
        hs = [vt.embeddings(x)]
        for layer in vt.encoder.layers:
            hs.append(layer(hs[-1], None))
        seq = vt.post_layernorm(hs[-1])
        if hasattr(m, "classifier"):
            pre = seq.mean(dim=1)
            logits = m.classifier(pre)
        else:
            pre = logits = vt.head(seq)
    model.float()
    return {"logits": logits.numpy(), "prelogits": pre.numpy(), "hidden_states": [h.numpy() for h in hs], "last_hidden_state": seq.numpy()}
