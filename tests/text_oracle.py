"""CLIP and SigLIP text towers for tests: tiny Hugging Face models as the float64 oracle, and the numpy emulation of the engine's text
schedule (vitb200_create_text).

The HF models are built from a config under torch.manual_seed with their weights redrawn by tests/hf_oracle.init_model (matrices
f16-valued, as the engine stores them), saved and converted with `convert.py --text`.  The emulation is tests/emulation.Emulation's
block loop on token rows instead of patch rows, with three additions: the token gather (f32(f16 table row) + pos_embed, no rounding),
the causal soft-max of CLIP (each query row's soft-max over keys 0 .. t alone, the reference's f16 soft-max on that prefix) and the
three pooling rules of vitb200_text_arch."""
import os

import numpy as np

from oracle import restatement as rs
from tests.emulation import Emulation
from tests.fp8_reference import _f16, e4m3_value, quantize_tensor
from tests.util import pkg

# name: (vocab, hidden, heads, layers, context, projection dim)
GEOMETRIES = {
    "micro": (1000, 128, 2, 2, 16, 96),
    "ctx77": (4000, 256, 4, 2, 77, 128),
    "siglip64": (2000, 128, 2, 2, 64, 128),
}
CLIP_ACT = {"quick_gelu": "quick_gelu", "gelu_erf": "gelu"}


def clip_text_config(geometry: str, activation: str = "quick_gelu", eos_token_id: int = 2):
    import transformers as tr
    V, D, H, L, N, E = GEOMETRIES[geometry]
    return tr.CLIPTextConfig(vocab_size=V, hidden_size=D, intermediate_size=4 * D, num_attention_heads=H, num_hidden_layers=L,
                             max_position_embeddings=N, hidden_act=CLIP_ACT[activation], layer_norm_eps=1e-5, projection_dim=E,
                             eos_token_id=eos_token_id, bos_token_id=0, pad_token_id=1, attn_implementation="eager")


def siglip_text_config(geometry: str = "siglip64"):
    import transformers as tr
    V, D, H, L, N, E = GEOMETRIES[geometry]
    return tr.SiglipTextConfig(vocab_size=V, hidden_size=D, intermediate_size=4 * D, num_attention_heads=H, num_hidden_layers=L,
                               max_position_embeddings=N, hidden_act="gelu_pytorch_tanh", layer_norm_eps=1e-6, projection_size=E,
                               attn_implementation="eager")


def build_clip(geometry: str = "micro", activation: str = "quick_gelu", eos_token_id: int = 2, projection: bool = True, seed: int = 0):
    """CLIPTextModelWithProjection (projection=True) or CLIPTextModel, float32, matrix weights f16-valued."""
    import transformers as tr
    from tests.hf_oracle import init_model
    cls = tr.CLIPTextModelWithProjection if projection else tr.CLIPTextModel
    return init_model(cls, clip_text_config(geometry, activation, eos_token_id), seed, norms=("layer_norm",), f32=("position_embedding",))


def build_siglip(geometry: str = "siglip64", seed: int = 0):
    import transformers as tr
    from tests.hf_oracle import init_model
    return init_model(tr.SiglipTextModel, siglip_text_config(geometry), seed, norms=("layer_norm",), f32=("position_embedding",))


def convert(model, directory: str, name: str = "text") -> str:
    """save_pretrained + `convert.py --text` -> the GGUF path."""
    model.save_pretrained(directory)
    out = os.path.join(directory, f"{name}.gguf")
    pkg.convert.main([os.path.join(directory, "model.safetensors"), out, "--hf-config", os.path.join(directory, "config.json"), "--text"])
    return out


def hf_outputs(model, ids) -> dict:
    """float64 oracle on ids [B][N]: embeds (text_embeds with a projection, pooler_output otherwise), pooled (last_hidden_state's pooled
    row: the head's input), hidden_states[i], i = 0 .. L, and last_hidden_state."""
    import torch
    m = model.double()
    with torch.no_grad():
        out = m(input_ids=torch.from_numpy(np.asarray(ids, np.int64)), output_hidden_states=True)
    model.float()
    emb = out.text_embeds if hasattr(out, "text_embeds") else out.pooler_output
    cfg = model.config
    rows = pool_rows(ids, "last" if "Siglip" in type(model).__name__ else ("eos_argmax" if cfg.eos_token_id == 2 else "eos"), cfg.eos_token_id)
    last = out.last_hidden_state.numpy()
    return {"embeds": emb.numpy(), "pooled": last[np.arange(len(rows)), rows],
            "hidden_states": [h.numpy() for h in out.hidden_states], "last_hidden_state": last}


def pool_rows(ids, pool: str, eos: int) -> np.ndarray:
    """The pooled row of each sequence under vitb200_text_arch.pool, first occurrence on ties (torch's argmax)."""
    ids = np.asarray(ids)
    if pool == "last":
        return np.full(len(ids), ids.shape[1] - 1)
    if pool == "eos_argmax":
        return ids.argmax(axis=1)
    hit = ids == eos
    return np.where(hit.any(axis=1), hit.argmax(axis=1), 0)


class TextEmulation(Emulation):
    """The f16 (fp8=False) or FP8 engine's text schedule on the host.  vf: a parsed text model file (ggml_file.VitFile with .text)."""

    def __init__(self, vf, acc=np.float32, fp8: bool = False):
        t = vf.tensors
        f32 = lambda n: np.asarray(t[n], np.float32).reshape(-1)
        self.acc, self.fp8, self.TH = acc, fp8, 1
        self.D, self.L, self.H, self.R = vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, 0
        self.activation, self.pool, self.text = vf.activation, "token", vf.text
        self.eps = float(vf.eps) if vf.eps else 1e-6
        self.tok = _f16(np.asarray(t["token_embd.weight"], np.float32))
        self.pos = f32("pos_embed").reshape(-1, self.D)
        self.blocks = []
        for i in range(self.L):
            p = f"blocks.{i}."
            blk = {k: f32(p + k) for k in ("norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "attn.qkv.bias", "attn.proj.bias",
                                          "mlp.fc1.bias", "mlp.fc2.bias")}
            for k in ("attn.qkv.weight", "attn.proj.weight", "mlp.fc1.weight", "mlp.fc2.weight"):
                w = np.asarray(t[p + k], np.float32).astype(np.float16)
                blk[k] = (e4m3_value(quantize_tensor(w)[0]), quantize_tensor(w)[1]) if fp8 and k in ("attn.qkv.weight", "mlp.fc1.weight") \
                    else w.astype(np.float32)
            self.blocks.append(blk)
        self.norm_w, self.norm_b = f32("norm.weight"), f32("norm.bias")
        self.w_head, self.b_head = _f16(np.asarray(t["head.weight"], np.float32)), f32("head.bias")

    def _softmax(self, s):
        """Soft-max of scores [B][H][N][N]; causal: row t over keys 0 .. t, the rest 0."""
        N = s.shape[-1]
        if not self.text["causal"]:
            return rs.softmax_rows(s.reshape(-1, N)).reshape(s.shape)
        p = np.zeros_like(s)
        for q in range(N):
            p[:, :, q, : q + 1] = rs.softmax_rows(np.ascontiguousarray(s[:, :, q, : q + 1]).reshape(-1, q + 1)).reshape(s.shape[:2] + (q + 1,))
        return p

    def encode_ids(self, ids, layers=None) -> np.ndarray:
        """ids [B][N] -> the residual stream [B][N][D] after `layers` blocks (None: all)."""
        ids = np.asarray(ids)
        B, N, D = ids.shape[0], ids.shape[1], self.D
        x = (self.tok[ids] + self.pos[None, :N]).reshape(B * N, D).astype(np.float32)
        for blk in self.blocks[:layers]:
            y = rs.layernorm(x, blk["norm1.weight"], blk["norm1.bias"], self.eps)
            qkv = self._ln_linear(y, blk["attn.qkv.weight"]) + blk["attn.qkv.bias"]
            qkv = qkv.reshape(B, N, 3, self.H, 64).transpose(2, 0, 3, 1, 4)
            s = np.einsum("bhqd,bhkd->bhqk", qkv[0].astype(self.acc), qkv[1].astype(self.acc)).astype(np.float32) * np.float32(0.125)
            p = self._softmax(s)
            o = np.einsum("bhqk,bhkd->bhqd", p.astype(self.acc), qkv[2].astype(self.acc)).astype(np.float32)
            o = _f16(o.transpose(0, 2, 1, 3).reshape(B * N, D))
            x = self._mm(o, blk["attn.proj.weight"]) + blk["attn.proj.bias"] + x
            y = rs.layernorm(x, blk["norm2.weight"], blk["norm2.bias"], self.eps)
            h = self._ln_linear(y, blk["mlp.fc1.weight"]) + blk["mlp.fc1.bias"]
            x = self._mm(self._act(h), blk["mlp.fc2.weight"]) + blk["mlp.fc2.bias"] + x
        return x.reshape(B, N, D)

    def pooled(self, ids, x) -> np.ndarray:
        """The final LayerNorm of each sequence's pooled row, f32 [B][D]."""
        rows = pool_rows(ids, self.text["pool"], self.text["eos_token_id"])
        return rs.layernorm(np.ascontiguousarray(np.asarray(x)[np.arange(len(rows)), rows]), self.norm_w, self.norm_b, self.eps)

    def embeds(self, ids) -> np.ndarray:
        """ids [B][N] -> embeds [B][E]: the head on f16(the pooled row)."""
        return self._mm(_f16(self.pooled(ids, self.encode_ids(ids))), self.w_head) + self.b_head


def padded_ids(rng, B: int, N: int, V: int, eos: int, eos_at, pad: int = 1) -> np.ndarray:
    """B sequences of N ids: random ids in [3, V) (not eos), eos at position eos_at[b] (None: no eos), random ids after it (padding that
    varies)."""
    ids = rng.integers(3, V, size=(B, N))
    ids[ids == eos] = 3
    for b, at in enumerate(eos_at):
        if at is not None:
            ids[b, at] = eos
    return ids.astype(np.int32)
