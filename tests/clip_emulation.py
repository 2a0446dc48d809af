"""The emulation of tests/fp8_reference.py (Fp8Emulation, f16 and FP8 forms) extended to a model file's architecture (vitb200_arch), for
tests of CLIP towers.

Everything Fp8Emulation holds is reused: the weights as the engine stores them, the e4m3 quantisation, the matrix products and the
restatement's LayerNorm, soft-max and GELU table.  What is added, taken from the VitFile:

    pre_norm    x = LayerNorm(x) (norm_pre.*, f32 in and out, the file's eps) on the embeddings, before block 0
    activation  gelu_tanh: f16(gelu_table(f16(h))) as before; gelu_erf / quick_gelu: f16(act(h)) on h itself, without rounding h to f16

The block schedule is Fp8Emulation.forward's, step for step, split into `encode` (the residual stream after any block, as
vitb200_features returns it) and `prelogits` (the final LayerNorm of the pooled rows).  On a reference-architecture file `forward` is
bit-identical to Fp8Emulation.forward (tests/test_clip.py checks this)."""
import numpy as np
from scipy.special import ndtr

from oracle import restatement as rs
from tests.fp8_reference import Fp8Emulation, _f16


class ArchEmulation(Fp8Emulation):
    """Fp8Emulation (fp8=True: the FP8 engine, fp8=False: the f16 engine) with the file's pre-norm and MLP activation."""

    def __init__(self, vf, head_tokens: int = 1, acc=np.float32, fp8: bool = True):
        super().__init__(vf, head_tokens, acc, fp8)
        f32 = lambda n: np.asarray(vf.tensors[n], np.float32).reshape(-1)
        self.eps = float(vf.eps) if getattr(vf, "eps", 0) else 1e-6
        self.pre_norm = (f32("norm_pre.weight"), f32("norm_pre.bias")) if getattr(vf, "pre_norm", 0) else None
        self.activation = getattr(vf, "activation", "gelu_tanh")

    def _act(self, h):
        """The fc1 epilogue's activation."""
        if self.activation == "gelu_tanh":
            return _f16(rs.gelu_table(_f16(h)))
        x = np.asarray(h, np.float64)
        if self.activation == "gelu_erf":
            return _f16(x * ndtr(x))                      # 0.5 x (1 + erf(x / sqrt 2))
        assert self.activation == "quick_gelu", self.activation
        with np.errstate(over="ignore"):
            return _f16(x / (1.0 + np.exp(-1.702 * x)))

    def encode(self, imgs, layers=None) -> np.ndarray:
        """imgs float32 [B][S][S][C] -> the residual stream [B][N][D] after `layers` blocks (None: all; 0: the input of block 0, after the
        pre-norm if the model has one)."""
        imgs = np.asarray(imgs, np.float32).reshape(-1, self.S, self.S, self.C)
        B, P, G, D = imgs.shape[0], self.P, self.S // self.P, self.D
        N = G * G + 1
        a = imgs.reshape(B, G, P, G, P, self.C).transpose(0, 1, 3, 5, 2, 4).reshape(B * G * G, -1)
        emb = (self._mm(_f16(a), self.w_patch) + self.b_patch).reshape(B, G * G, D) + self.pos[1:]
        x = np.concatenate([np.broadcast_to(self.cls + self.pos[0], (B, 1, D)), emb], axis=1).reshape(B * N, D).astype(np.float32)
        eps = self.eps
        if self.pre_norm is not None:
            x = rs.layernorm(x, *self.pre_norm, eps)
        for blk in self.blocks[: self.L if layers is None else layers]:
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
            x = (self._mm(self._act(h), blk["mlp.fc2.weight"]) + blk["mlp.fc2.bias"]) + x
        return x.reshape(B, N, D)

    def prelogits(self, x) -> np.ndarray:
        """The residual stream [B][N][D] -> the final LayerNorm of the head_tokens pooled rows, f32 [B * head_tokens][D]."""
        pooled = np.asarray(x, np.float32)[:, : self.TH].reshape(-1, self.D)
        return rs.layernorm(pooled, self.norm_w, self.norm_b, self.eps)

    def forward(self, imgs) -> np.ndarray:
        """Logits [B][num_classes] ([B][head_tokens][num_classes]), as Fp8Emulation.forward returns them."""
        x = self.encode(imgs)
        logits = self._mm(_f16(self.prelogits(x)), self.w_head) + self.b_head
        return logits.reshape(x.shape[0], -1) if self.TH == 1 else logits.reshape(x.shape[0], self.TH, -1)
