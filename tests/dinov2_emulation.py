"""The emulation of tests/clip_emulation.py (ArchEmulation, f16 and FP8 forms) extended to DINOv2's architecture, for tests.

What is added, taken from the VitFile:

    layer_scale  x = f32(f32(proj(o) + b) * gamma1) + x and likewise for fc2 with gamma2: the engine's LayerScale epilogue order
    reg_tokens   rows 1 .. R of every image are reg_token[r] + pos_embed[1 + r]; the patches follow at rows 1 + R ..
    pool         cls_patch_mean: the head reads [LN(row 0) || mean over the patch rows of LN(row)], the registers left out

On a file without these keys every method is ArchEmulation's, bit for bit (tests/test_dinov2.py checks this)."""
import numpy as np

from oracle import restatement as rs
from tests.clip_emulation import ArchEmulation
from tests.fp8_reference import _f16


class DinoEmulation(ArchEmulation):
    """ArchEmulation with LayerScale, register tokens and the class-plus-patch-mean pool."""

    def __init__(self, vf, head_tokens: int = 1, acc=np.float32, fp8: bool = True):
        super().__init__(vf, head_tokens, acc, fp8)
        f32 = lambda n: np.asarray(vf.tensors[n], np.float32).reshape(-1)
        self.R = int(getattr(vf, "reg_tokens", 0))
        self.reg = f32("reg_token").reshape(self.R, self.D) if self.R else np.zeros((0, self.D), np.float32)
        self.pool = getattr(vf, "pool", "token")
        self.gammas = [(f32(f"blocks.{i}.ls1.gamma"), f32(f"blocks.{i}.ls2.gamma")) if getattr(vf, "layer_scale", 0) else None
                       for i in range(self.L)]

    def encode(self, imgs, layers=None) -> np.ndarray:
        """The residual stream [B][N][D] after `layers` blocks, rows [cls, registers, patches]."""
        if not self.R and not any(self.gammas):
            return super().encode(imgs, layers)
        imgs = np.asarray(imgs, np.float32).reshape(-1, self.S, self.S, self.C)
        B, P, G, D, R = imgs.shape[0], self.P, self.S // self.P, self.D, self.R
        N = G * G + 1 + R
        a = imgs.reshape(B, G, P, G, P, self.C).transpose(0, 1, 3, 5, 2, 4).reshape(B * G * G, -1)
        emb = (self._mm(_f16(a), self.w_patch) + self.b_patch).reshape(B, G * G, D) + self.pos[1 + R:]
        prefix = np.concatenate([self.cls[None], self.reg]) + self.pos[: 1 + R]
        x = np.concatenate([np.broadcast_to(prefix, (B, 1 + R, D)), emb], axis=1).reshape(B * N, D).astype(np.float32)
        eps = self.eps
        if self.pre_norm is not None:
            x = rs.layernorm(x, *self.pre_norm, eps)
        for blk, g in list(zip(self.blocks, self.gammas))[: self.L if layers is None else layers]:
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
            br = self._mm(o, blk["attn.proj.weight"]) + blk["attn.proj.bias"]
            x = (br * g[0] if g else br) + x
            y = rs.layernorm(x, blk["norm2.weight"], blk["norm2.bias"], eps)
            if self.fp8:
                h = self._fp8_linear(y, blk["mlp.fc1.weight"]) + blk["mlp.fc1.bias"]
            else:
                h = self._mm(_f16(y), blk["mlp.fc1.weight"]) + blk["mlp.fc1.bias"]
            br = self._mm(self._act(h), blk["mlp.fc2.weight"]) + blk["mlp.fc2.bias"]
            x = (br * g[1] if g else br) + x
        return x.reshape(B, N, D)

    def prelogits(self, x, norm: bool = True) -> np.ndarray:
        """The head's input, f32: [B * head_tokens][D], or [B][2 D] for the cls_patch_mean pool (norm = False: without the LayerNorm)."""
        if self.pool != "cls_patch_mean":
            return super().prelogits(x)
        x = np.asarray(x, np.float32)
        B, N, D = x.shape
        y = rs.layernorm(x.reshape(-1, D), self.norm_w, self.norm_b, self.eps).reshape(B, N, D) if norm else x
        return np.concatenate([y[:, 0], y[:, 1 + self.R:].astype(np.float64).mean(axis=1).astype(np.float32)], axis=1)

    def forward(self, imgs) -> np.ndarray:
        if self.pool != "cls_patch_mean":
            return super().forward(imgs)
        return self._mm(_f16(self.prelogits(self.encode(imgs))), self.w_head) + self.b_head
