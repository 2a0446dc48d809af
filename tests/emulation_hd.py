"""tests/emulation.py's forward pass for any head dim, for tests of models whose attention heads are not 64 columns wide (ViT-H/14: 80).

The one difference is in the attention: q, k and v are split into heads of hd = D / H columns, and the scores are scaled by the
reference's 1 / sqrtf(hd) in f32 (vit.cpp:854), which is 0.125 at hd = 64.  Everything else -- the f16 and FP8 forms, the architectures,
the pools and the head -- is tests.emulation.Emulation's, which forward() and prelogits() reach through encode()."""
import numpy as np

from oracle import restatement as rs
from tests import emulation as base
from tests.fp8_reference import _f16


class Emulation(base.Emulation):
    """base.Emulation with the head split by D // H and the scale 1 / sqrtf(hd)."""

    def encode(self, imgs, layers=None) -> np.ndarray:
        """As base.Emulation.encode: imgs float32 [B][S][S][C] -> the residual stream [B][N][D] after `layers` blocks."""
        imgs = np.asarray(imgs, np.float32).reshape(-1, self.S, self.S, self.C)
        B, P, G, D, eps = imgs.shape[0], self.P, self.S // self.P, self.D, self.eps
        hd = D // self.H
        scale = np.float32(1) / np.sqrt(np.float32(hd))
        n0 = len(self.prefix)
        N = n0 + G * G
        a = imgs.reshape(B, G, P, G, P, self.C).transpose(0, 1, 3, 5, 2, 4).reshape(B * G * G, -1)
        emb = (self._mm(_f16(a), self.w_patch) + self.b_patch).reshape(B, G * G, D) + self.pos[n0:]
        x = np.concatenate([np.broadcast_to(self.prefix, (B, n0, D)), emb], axis=1).reshape(B * N, D).astype(np.float32)
        if self.pre_norm is not None:
            x = rs.layernorm(x, *self.pre_norm, eps)
        for blk in self.blocks[:layers]:
            y = rs.layernorm(x, blk["norm1.weight"], blk["norm1.bias"], eps)
            qkv = self._ln_linear(y, blk["attn.qkv.weight"]) + blk["attn.qkv.bias"]
            qkv = qkv.reshape(B, N, 3, self.H, hd).transpose(2, 0, 3, 1, 4)  # [3][B][H][N][hd]
            s = np.einsum("bhqd,bhkd->bhqk", qkv[0].astype(self.acc), qkv[1].astype(self.acc)).astype(np.float32) * scale
            p = rs.softmax_rows(s.reshape(-1, N)).reshape(s.shape)
            o = np.einsum("bhqk,bhkd->bhqd", p.astype(self.acc), qkv[2].astype(self.acc)).astype(np.float32)
            o = _f16(o.transpose(0, 2, 1, 3).reshape(B * N, D))
            br = self._mm(o, blk["attn.proj.weight"]) + blk["attn.proj.bias"]
            x = (br * blk["ls1.gamma"] if "ls1.gamma" in blk else br) + x
            y = rs.layernorm(x, blk["norm2.weight"], blk["norm2.bias"], eps)
            h = self._ln_linear(y, blk["mlp.fc1.weight"]) + blk["mlp.fc1.bias"]
            br = self._mm(self._act(h), blk["mlp.fc2.weight"]) + blk["mlp.fc2.bias"]
            x = (br * blk["ls2.gamma"] if "ls2.gamma" in blk else br) + x
        return x.reshape(B, N, D)
