"""Numpy emulation of the FP8 engine's recipe (vitb200_create_fp8, numerics in include/vitb200.h), for tests.

The f16 engine's forward pass as the restatement (oracle/restatement.py) defines its pieces -- LayerNorm, the f16 rounding of every
GEMM's A operand and weights, the reference's soft-max and GELU tables -- with qkv and fc1 replaced by the FP8 form:

    y   = LayerNorm(x)                      f32, per token row
    sa  = amax(|y|) / 448,  qa = e4m3(y * (448 / amax))          (scale 1 for an all-zero row)
    sw  = amax(|w16|) / 448, qw = e4m3(w16 * (448 / amax))       (per tensor)
    out = sum_k qa qw * (sa * sw) + bias                         then the f16 engine's epilogue (qkv: f32; fc1: f16, GELU, f16)

q, k and v stay f32 (the engine carries them as hi + lo f16 pairs, ~22 bits).  `acc` selects the accumulation type of every matrix
product: float32 is what the GPU does (to within the order of the sum), float64 the floor against which the f32 rounding noise of
the emulation itself is measured."""
import numpy as np
import torch

from oracle import restatement as rs

E4M3_MAX = np.float32(448.0)


def e4m3_bits(x) -> np.ndarray:
    """f32 -> e4m3 bytes, round to nearest even (torch saturates nothing: callers keep |x| <= 448)."""
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def e4m3_value(bits) -> np.ndarray:
    """e4m3 bytes -> their f32 values."""
    return torch.from_numpy(np.ascontiguousarray(bits, np.uint8)).view(torch.float8_e4m3fn).to(torch.float32).numpy()


def _scales(amax):
    amax = np.asarray(amax, np.float32)
    nz = amax > 0
    safe = np.where(nz, amax, np.float32(1))
    inv = np.where(nz, E4M3_MAX / safe, np.float32(1)).astype(np.float32)
    sc = np.where(nz, safe / E4M3_MAX, np.float32(1)).astype(np.float32)
    return inv, sc


def quantize_rows(y):
    """y float32 [R][K] -> (e4m3 bytes [R][K], scales float32 [R]): the FP8 engine's LayerNorm output."""
    y = np.ascontiguousarray(y, np.float32)
    inv, sc = _scales(np.abs(y).max(axis=1))
    return e4m3_bits(y * inv[:, None]), sc


def quantize_tensor(w16):
    """f16 weights -> (e4m3 bytes, f32 scale): the FP8 engine's upload-time quantisation."""
    w = np.asarray(w16, np.float16).astype(np.float32)
    inv, sc = _scales(np.abs(w).max() if w.size else 0.0)
    return e4m3_bits(w * inv), np.float32(sc)


def _f16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


class Fp8Emulation:
    """The FP8 (fp8=True) or f16 (fp8=False) engine's forward pass on the host.  vf: a parsed model file (ggml_file.VitFile)."""

    def __init__(self, vf, head_tokens: int = 1, acc=np.float32, fp8: bool = True):
        self.vf, self.acc, self.fp8, self.TH = vf, acc, fp8, head_tokens
        t = vf.tensors
        self.D, self.L, self.H = vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads
        self.P, self.S = vf.patch_size, vf.img_size
        pw = np.asarray(t["patch_embed.proj.weight"], np.float32)
        self.C = pw.shape[1]
        self.w_patch = _f16(pw.reshape(self.D, -1))
        f32 = lambda n: np.asarray(t[n], np.float32).reshape(-1)
        self.b_patch, self.cls, self.pos = f32("patch_embed.proj.bias"), f32("cls_token"), f32("pos_embed").reshape(-1, self.D)
        self.blocks = []
        for i in range(self.L):
            p = f"blocks.{i}."
            blk = {k: f32(p + k) for k in ("norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "attn.qkv.bias",
                                           "attn.proj.bias", "mlp.fc1.bias", "mlp.fc2.bias")}
            for k in ("attn.qkv.weight", "attn.proj.weight", "mlp.fc1.weight", "mlp.fc2.weight"):
                w16 = np.asarray(t[p + k], np.float32).astype(np.float16)
                if fp8 and k in ("attn.qkv.weight", "mlp.fc1.weight"):
                    q, sc = quantize_tensor(w16)
                    blk[k] = (e4m3_value(q), sc)
                else:
                    blk[k] = w16.astype(np.float32)
            self.blocks.append(blk)
        self.norm_w, self.norm_b = f32("norm.weight"), f32("norm.bias")
        self.w_head, self.b_head = _f16(np.asarray(t["head.weight"], np.float32)), f32("head.bias")

    def _mm(self, a, w):
        return (a.astype(self.acc) @ w.astype(self.acc).T).astype(np.float32)

    def _fp8_linear(self, y, wq):
        qw, sw = wq
        qa, sa = quantize_rows(y)
        acc = self._mm(e4m3_value(qa), qw)
        return acc * (sa * sw)[:, None]

    def forward(self, imgs) -> np.ndarray:
        """imgs float32 [B][S][S][C] (or [B][S][S] for one channel) -> logits [B][num_classes] ([B][head_tokens][num_classes])."""
        imgs = np.asarray(imgs, np.float32).reshape(-1, self.S, self.S, self.C)
        B, P, G, D = imgs.shape[0], self.P, self.S // self.P, self.D
        N = G * G + 1
        # im2col, k = c*P*P + ky*P + kx, rounded to f16
        a = imgs.reshape(B, G, P, G, P, self.C).transpose(0, 1, 3, 5, 2, 4).reshape(B * G * G, -1)
        emb = (self._mm(_f16(a), self.w_patch) + self.b_patch).reshape(B, G * G, D) + self.pos[1:]
        x = np.concatenate([np.broadcast_to(self.cls + self.pos[0], (B, 1, D)), emb], axis=1).reshape(B * N, D).astype(np.float32)
        eps = float(self.vf.eps) if getattr(self.vf, "eps", 0) else 1e-6
        for blk in self.blocks:
            y = rs.layernorm(x, blk["norm1.weight"], blk["norm1.bias"], eps)
            if self.fp8:
                qkv = self._fp8_linear(y, blk["attn.qkv.weight"]) + blk["attn.qkv.bias"]
            else:
                qkv = self._mm(_f16(y), blk["attn.qkv.weight"]) + blk["attn.qkv.bias"]
            qkv = qkv.reshape(B, N, 3, self.H, 64).transpose(2, 0, 3, 1, 4)  # [3][B][H][N][64]
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
            h = _f16(rs.gelu_table(_f16(h)))
            x = (self._mm(h, blk["mlp.fc2.weight"]) + blk["mlp.fc2.bias"]) + x
        pooled = x.reshape(B, N, D)[:, : self.TH].reshape(B * self.TH, D)
        f = _f16(rs.layernorm(pooled, self.norm_w, self.norm_b, eps))
        logits = self._mm(f, self.w_head) + self.b_head
        return logits.reshape(B, -1) if self.TH == 1 else logits.reshape(B, self.TH, -1)


def rel_dist(a, b) -> np.ndarray:
    """Per image max|a - b| / max|b| over the last axis (and the token axis, if any)."""
    a = np.asarray(a, np.float64).reshape(a.shape[0], -1)
    b = np.asarray(b, np.float64).reshape(b.shape[0], -1)
    return np.abs(a - b).max(axis=1) / np.abs(b).max(axis=1)
