"""SigLIP So400m-shaped towers for tests: 72-column attention heads, MLP widths that are not 4 D and image sizes the patch does not
divide, as Hugging Face float64 oracles and the emulation of the engine's forward pass.

The models are tests/siglip_oracle.py's and tests/text_oracle.py's (seeded, weights redrawn by tests/hf_oracle.init_model, saved and
converted with convert.py), built from the geometries below with 2 layers.  The emulation is tests/emulation_hd.py's with what these
towers add: the patch matrix from the top-left G P x G P pixels (G = floor(img_size / patch), as HF's valid conv takes them) and the
attention-pooling head split into heads of D / H columns with the scale f32(1 / sqrtf(hd))."""
import numpy as np

from tests import emulation_hd
from tests.fp8_reference import _f16
from tests.hf_oracle import init_model

# name: (hidden, heads, MLP width, patch, image size)
GEOMETRIES = {
    "micro72": (144, 2, 576, 16, 64),          # 16 tokens, F = 4 D: the split-precision form
    "micro72_p14": (144, 2, 464, 14, 64),      # 16 tokens, F not 4 D, 8 pixel rows and columns dropped
    "so400m_224": (1152, 16, 4304, 14, 224),   # 256 tokens: the f16 form
    "so400m_384": (1152, 16, 4304, 14, 384),   # 729 tokens, 6 pixel rows and columns dropped
}
LAYERS = 2
NUM_LABELS = 10
# text: (vocab, hidden, heads, MLP width, context, projection)
TEXT = (500, 1152, 16, 4304, 64, 1152)


def vision_config(geometry: str):
    import transformers as tr
    D, H, F, P, S = GEOMETRIES[geometry]
    return tr.SiglipVisionConfig(hidden_size=D, intermediate_size=F, num_attention_heads=H, num_hidden_layers=LAYERS, patch_size=P,
                                 image_size=S, hidden_act="gelu_pytorch_tanh", layer_norm_eps=1e-6, attn_implementation="eager")


def text_config():
    import transformers as tr
    V, D, H, F, N, E = TEXT
    return tr.SiglipTextConfig(vocab_size=V, hidden_size=D, intermediate_size=F, num_attention_heads=H, num_hidden_layers=LAYERS,
                               max_position_embeddings=N, hidden_act="gelu_pytorch_tanh", layer_norm_eps=1e-6, projection_size=E,
                               attn_implementation="eager")


def build_hf(geometry: str, classifier: bool = False, seed: int = 0):
    """SiglipForImageClassification (classifier) or SiglipVisionModel, float32, matrix weights f16-valued."""
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


def build_text(seed: int = 0):
    import transformers as tr
    return init_model(tr.SiglipTextModel, text_config(), seed, norms=("layer_norm",), f32=("position_embedding",))


def build_clip_pair(geometry: str = "micro72", seed: int = 0):
    """A SiglipModel with a So400m-shaped image tower (`geometry`) and text tower (TEXT, projection = the image width)."""
    import transformers as tr
    tc = text_config().to_dict()
    D = GEOMETRIES[geometry][0]
    tc.update(hidden_size=D, num_attention_heads=GEOMETRIES[geometry][1], intermediate_size=GEOMETRIES[geometry][2], projection_size=D)
    cfg = tr.SiglipConfig(vision_config=vision_config(geometry).to_dict(), text_config=tc)
    cfg._attn_implementation = "eager"
    return init_model(tr.SiglipModel, cfg, seed, norms=("norm",), f32=("position_embedding", "probe"))


class Emulation(emulation_hd.Emulation):
    """emulation_hd.Emulation with the floor grid and the head-dim-hd attention-pooling head.  crop: the pixel window the patches are
    read from, (top, left) of a G P x G P square; (0, 0) is what HF and the engine do."""

    def __init__(self, vf, crop=(0, 0), **kw):
        super().__init__(vf, **kw)
        self.crop = crop

    def encode(self, imgs, layers=None) -> np.ndarray:
        S, GP = self.S, self.S // self.P * self.P
        y, x = self.crop
        imgs = np.asarray(imgs, np.float32).reshape(-1, S, S, self.C)[:, y:y + GP, x:x + GP]
        self.S = GP
        try:
            return super().encode(imgs, layers)
        finally:
            self.S = S

    def pool_attention(self, y) -> np.ndarray:
        B, N, D = y.shape
        H = self.H
        hd = D // H
        kv = _f16(self._mm(_f16(y.reshape(-1, D)), self.w_kv) + self.b_kv).reshape(B, N, 2, H, hd)
        k, v = kv[:, :, 0].transpose(0, 2, 1, 3), kv[:, :, 1].transpose(0, 2, 1, 3)
        q = (self.q * (np.float32(1) / np.sqrt(np.float32(hd)))).reshape(H, hd)
        s = np.einsum("hd,bhnd->bhn", q.astype(self.acc), k.astype(self.acc)).astype(np.float32)
        e = np.exp((s - s.max(axis=2, keepdims=True)).astype(np.float64)).astype(np.float32)
        o = np.einsum("bhn,bhnd->bhd", e.astype(self.acc), v.astype(self.acc)) / e.astype(self.acc).sum(axis=2)[..., None]
        o = _f16(np.asarray(o, np.float32).reshape(B, D))
        return self._mm(o, self.w_pp) + self.b_pp


def attention_ref(qkv, B, N, H, hd):
    """float64 attention of row-major q | k | v [B*N][3 H hd] -> [B*N][H hd]."""
    x = np.asarray(qkv, np.float64).reshape(B, N, 3, H, hd).transpose(2, 0, 3, 1, 4)
    s = np.einsum("bhqd,bhkd->bhqk", x[0], x[1]) / np.sqrt(hd)
    p = np.exp(s - s.max(axis=3, keepdims=True))
    p /= p.sum(axis=3, keepdims=True)
    return np.einsum("bhqk,bhkd->bhqd", p, x[2]).transpose(0, 2, 1, 3).reshape(B * N, H * hd)


def pool_ref(q, kv, B, P, H, hd=72):
    """float64 probe attention: q [H hd], kv [B*P][2 H hd] (rows k then v) -> [B][H hd]."""
    kv = np.asarray(kv, np.float64).reshape(B, P, 2, H, hd)
    s = np.einsum("hd,bphd->bhp", np.asarray(q, np.float64).reshape(H, hd), kv[:, :, 0]) / np.sqrt(hd)
    p = np.exp(s - s.max(axis=2, keepdims=True))
    p /= p.sum(axis=2, keepdims=True)
    return np.einsum("bhp,bphd->bhd", p, kv[:, :, 1]).reshape(B, H * hd)
