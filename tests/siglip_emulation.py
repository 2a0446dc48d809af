"""The emulation of tests/dinov2_emulation.py (DinoEmulation, f16 and FP8 forms) extended to SigLIP's architecture, for tests.

What is added, taken from the VitFile:

    pool map / mean    no class token: the token rows are the patches, row p = patch(p) + pos_embed[p]
    pool map           the attention-pooling head, as the engine schedules it: y = f16(LN(rows)) (the final LayerNorm); k | v =
                       f16(y Wkv^T + bkv); per head softmax(q k / 8) over the image's rows in f32 with q = f32(latent Wq^T + bq) (f64);
                       o = f16(sum p v); h = o Wproj^T + bproj (f32); pooled = h + f16(act(f16(LN_head(h)) Wfc1^T + b)) Wfc2^T + b
    pool mean          the mean over all rows of LN(row)
    gelu_pytorch_tanh  f16(0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))) on the f32 x itself

On a file without these keys every method is DinoEmulation's, bit for bit (tests/test_siglip.py checks this)."""
import copy

import numpy as np

from oracle import restatement as rs
from tests.dinov2_emulation import DinoEmulation
from tests.fp8_reference import _f16
from tests.util import gf


def gelu_pytorch_tanh(x):
    x = np.asarray(x, np.float64)
    return 0.5 * x * (1.0 + np.tanh(np.sqrt(2.0 / np.pi) * (x + 0.044715 * x ** 3)))


class SiglipEmulation(DinoEmulation):
    """DinoEmulation with patch-only token rows, the attention-pooling head, the mean pool and PyTorch's tanh GELU."""

    def __init__(self, vf, head_tokens: int = 1, acc=np.float32, fp8: bool = True):
        self.patch_only = getattr(vf, "pool", "token") in gf.PATCH_ONLY_POOLS
        if self.patch_only:
            # the parent classes read a class token: give them a zero one, never used below
            vf = copy.copy(vf)
            vf.tensors = dict(vf.tensors, cls_token=np.zeros((1, 1, vf.hidden_size), np.float32))
        super().__init__(vf, head_tokens, acc, fp8)
        if getattr(vf, "pool", "token") == "map":
            t, D = vf.tensors, self.D
            f32 = lambda n: np.asarray(t[n], np.float32).reshape(-1)
            w16 = lambda n: _f16(np.asarray(t[n], np.float32))
            lat = np.asarray(t["attn_pool.latent"], np.float64).reshape(D)
            self.q = (np.asarray(t["attn_pool.q.weight"], np.float64) @ lat + np.asarray(t["attn_pool.q.bias"], np.float64)).astype(np.float32)
            self.w_kv, self.b_kv = w16("attn_pool.kv.weight"), f32("attn_pool.kv.bias")
            self.w_pp, self.b_pp = w16("attn_pool.proj.weight"), f32("attn_pool.proj.bias")
            self.pn_w, self.pn_b = f32("attn_pool.norm.weight"), f32("attn_pool.norm.bias")
            self.w_f1, self.b_f1 = w16("attn_pool.mlp.fc1.weight"), f32("attn_pool.mlp.fc1.bias")
            self.w_f2, self.b_f2 = w16("attn_pool.mlp.fc2.weight"), f32("attn_pool.mlp.fc2.bias")

    def _act(self, h):
        if self.activation == "gelu_pytorch_tanh":
            return _f16(gelu_pytorch_tanh(h))
        return super()._act(h)

    def encode(self, imgs, layers=None) -> np.ndarray:
        """The residual stream [B][N][D] after `layers` blocks; N = P patch rows for pools map / mean."""
        if not self.patch_only:
            return super().encode(imgs, layers)
        imgs = np.asarray(imgs, np.float32).reshape(-1, self.S, self.S, self.C)
        B, P, G, D = imgs.shape[0], self.P, self.S // self.P, self.D
        N = G * G
        a = imgs.reshape(B, G, P, G, P, self.C).transpose(0, 1, 3, 5, 2, 4).reshape(B * G * G, -1)
        x = ((self._mm(_f16(a), self.w_patch) + self.b_patch).reshape(B, N, D) + self.pos).reshape(B * N, D).astype(np.float32)
        eps = self.eps
        for blk in self.blocks[: self.L if layers is None else layers]:
            y = rs.layernorm(x, blk["norm1.weight"], blk["norm1.bias"], eps)
            if self.fp8:
                qkv = self._fp8_linear(y, blk["attn.qkv.weight"]) + blk["attn.qkv.bias"]
            else:
                qkv = self._mm(_f16(y), blk["attn.qkv.weight"]) + blk["attn.qkv.bias"]
            qkv = qkv.reshape(B, N, 3, self.H, 64).transpose(2, 0, 3, 1, 4)
            s = np.einsum("bhqd,bhkd->bhqk", qkv[0].astype(self.acc), qkv[1].astype(self.acc)).astype(np.float32) * np.float32(0.125)
            p = rs.softmax_rows(s.reshape(-1, N)).reshape(s.shape)
            o = np.einsum("bhqk,bhkd->bhqd", p.astype(self.acc), qkv[2].astype(self.acc)).astype(np.float32)
            o = _f16(o.transpose(0, 2, 1, 3).reshape(B * N, D))
            x = (self._mm(o, blk["attn.proj.weight"]) + blk["attn.proj.bias"]) + x
            y = rs.layernorm(x, blk["norm2.weight"], blk["norm2.bias"], eps)
            if self.fp8:
                h = self._fp8_linear(y, blk["mlp.fc1.weight"]) + blk["mlp.fc1.bias"]
            else:
                h = self._mm(_f16(y), blk["mlp.fc1.weight"]) + blk["mlp.fc1.bias"]
            x = (self._mm(self._act(h), blk["mlp.fc2.weight"]) + blk["mlp.fc2.bias"]) + x
        return x.reshape(B, N, D)

    def final_ln(self, x) -> np.ndarray:
        x = np.asarray(x, np.float32)
        B, N, D = x.shape
        return rs.layernorm(x.reshape(-1, D), self.norm_w, self.norm_b, self.eps).reshape(B, N, D)

    def pool_attention(self, y) -> np.ndarray:
        """The probe's attention over the final LayerNorm's rows y [B][N][D] (f32) and out_proj: h [B][D], f32."""
        B, N, D = y.shape
        H = self.H
        kv = _f16(self._mm(_f16(y.reshape(-1, D)), self.w_kv) + self.b_kv).reshape(B, N, 2, H, 64)
        k, v = kv[:, :, 0].transpose(0, 2, 1, 3), kv[:, :, 1].transpose(0, 2, 1, 3)      # [B][H][N][64]
        q = (self.q * np.float32(0.125)).reshape(H, 64)
        s = np.einsum("hd,bhnd->bhn", q.astype(self.acc), k.astype(self.acc)).astype(np.float32)
        e = np.exp((s - s.max(axis=2, keepdims=True)).astype(np.float64)).astype(np.float32)
        o = np.einsum("bhn,bhnd->bhd", e.astype(self.acc), v.astype(self.acc)) / e.astype(self.acc).sum(axis=2)[..., None]
        o = _f16(np.asarray(o, np.float32).reshape(B, D))
        return self._mm(o, self.w_pp) + self.b_pp

    def head_mlp(self, h) -> np.ndarray:
        """The head's MLP branch on h [B][D]: fc2(act(fc1(f16(LN_head(h))))), f32."""
        z = _f16(rs.layernorm(h, self.pn_w, self.pn_b, self.eps))
        return self._mm(self._act(self._mm(z, self.w_f1) + self.b_f1), self.w_f2) + self.b_f2

    def map_head(self, y) -> np.ndarray:
        """The attention-pooling head on the final LayerNorm's rows y [B][N][D] (f32) -> the pooled rows [B][D], f32."""
        h = self.pool_attention(y)
        return self.head_mlp(h) + h

    def prelogits(self, x, norm: bool = True) -> np.ndarray:
        """The head's input, f32 [B][D]: the attention-pooling head's row (map; needs the norm) or the mean of the rows (mean), through the
        final LayerNorm first when `norm`."""
        if not self.patch_only:
            return super().prelogits(x, norm) if self.pool == "cls_patch_mean" else super().prelogits(x)
        y = self.final_ln(x) if norm else np.asarray(x, np.float32)
        if self.pool == "map":
            assert norm, "the attention-pooling head reads the final LayerNorm's rows"
            return self.map_head(y)
        return y.astype(np.float64).mean(axis=1).astype(np.float32)

    def forward(self, imgs) -> np.ndarray:
        if not self.patch_only:
            return super().forward(imgs)
        return self._mm(_f16(self.prelogits(self.encode(imgs))), self.w_head) + self.b_head
