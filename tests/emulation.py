"""Numpy emulation of the engine's forward pass, f16 and FP8 forms, for every architecture a model file describes (vitb200_arch), for
tests.

The f16 engine's forward pass as the restatement (oracle/restatement.py) defines its pieces -- LayerNorm, the f16 rounding of every
GEMM's A operand and weights, the reference's soft-max and GELU tables.  The FP8 form (fp8=True, vitb200_create_fp8) runs qkv and fc1 on
e4m3 operands, quantised as tests/fp8_reference.py describes; every other GEMM stays f16.  q, k and v stay f32 (the engine carries them
as hi + lo f16 pairs, ~22 bits).  `acc` selects the accumulation type of every matrix product: float32 is what the GPU does (to within
the order of the sum), float64 the floor against which the f32 rounding noise of the emulation itself is measured.

The architecture comes from the VitFile's fields:

    pre_norm     x = LayerNorm(x) (norm_pre.*, f32 in and out, the file's eps) on the embeddings, before block 0
    activation   the fc1 epilogue's, from ACTIVATIONS on h = f32(acc + bias), rounded to f16: gelu_tanh is the reference's f16 table on
                 f16(h); the others are computed in float64 on h itself
    layer_scale  x = f32(f32(proj(o) + b) * gamma1) + x and likewise for fc2 with gamma2: the engine's LayerScale epilogue order
    reg_tokens   rows 1 .. R of every image are reg_token[r] + pos_embed[1 + r]; the patches follow at rows 1 + R ..
    pool         token           the final LayerNorm of the first head_tokens rows (25 for ViTSTR)
                 cls_patch_mean  [LN(row 0) || mean over the patch rows of LN(row)], the registers left out
                 map / mean      no class token: the token rows are the patches, row p = patch(p) + pos_embed[p]
                 map             the attention-pooling head, as the engine schedules it: y = LN(rows) (the final LayerNorm); k | v =
                                 f16(f16(y) Wkv^T + bkv); per head softmax(q k / 8) over the image's rows in f32 with q = f32(latent Wq^T +
                                 bq) (f64); o = f16(sum p v); h = o Wproj^T + bproj (f32); pooled = h + fc2(act(f16(LN_head(h)) Wfc1^T + b))
                 mean            the mean over all rows of LN(row)"""
import numpy as np
from scipy.special import ndtr

from oracle import restatement as rs
from tests.fp8_reference import _f16, e4m3_value, quantize_rows, quantize_tensor
from tests.util import gf


def gelu_pytorch_tanh(x):
    x = np.asarray(x, np.float64)
    return 0.5 * x * (1.0 + np.tanh(np.sqrt(2.0 / np.pi) * (x + 0.044715 * x ** 3)))


def _swiglu(x):
    """silu(x1) * x2, x1 | x2 the two halves of fc1's output (its rows in HF's order), silu(x) = x / (1 + e^-x)."""
    x1, x2 = np.split(x, 2, axis=-1)
    return x1 / (1.0 + np.exp(-x1)) * x2


# vitb200_arch.activation -> the fc1 epilogue's activation on x, float64 values of h = f32(acc + bias), before the f16 rounding
ACTIVATIONS = {
    "gelu_tanh": lambda x: rs.gelu_table(_f16(x)),
    "gelu_erf": lambda x: x * ndtr(x),                     # 0.5 x (1 + erf(x / sqrt 2))
    "quick_gelu": lambda x: x / (1.0 + np.exp(-1.702 * x)),
    "gelu_pytorch_tanh": gelu_pytorch_tanh,
    "swiglu": _swiglu,
}
assert tuple(ACTIVATIONS) == gf.ARCH_ACTIVATIONS


class Emulation:
    """The FP8 (fp8=True) or f16 (fp8=False) engine's forward pass on the host.  vf: a parsed model file (ggml_file.VitFile)."""

    def __init__(self, vf, head_tokens: int = 1, acc=np.float32, fp8: bool = True):
        assert head_tokens == 1 or vf.pool == "token", (head_tokens, vf.pool)
        self.acc, self.fp8, self.TH = acc, fp8, head_tokens
        t = vf.tensors
        f32 = lambda n: np.asarray(t[n], np.float32).reshape(-1)
        w16 = lambda n: _f16(np.asarray(t[n], np.float32))
        self.D, self.L, self.H, self.R = vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.reg_tokens
        self.P, self.S, self.pool, self.activation = vf.patch_size, vf.img_size, vf.pool, vf.activation
        D, R = self.D, self.R
        self.eps = float(vf.eps) if vf.eps else 1e-6
        self.pre_norm = (f32("norm_pre.weight"), f32("norm_pre.bias")) if vf.pre_norm else None
        pw = np.asarray(t["patch_embed.proj.weight"], np.float32)
        self.C = pw.shape[1]
        self.w_patch, self.b_patch, self.pos = _f16(pw.reshape(D, -1)), f32("patch_embed.proj.bias"), f32("pos_embed").reshape(-1, D)
        # the rows ahead of the patches, with their positions: the class token and the registers, or none
        if self.pool in gf.PATCH_ONLY_POOLS:
            self.prefix = np.zeros((0, D), np.float32)
        else:
            reg = f32("reg_token").reshape(R, D) if R else np.zeros((0, D), np.float32)
            self.prefix = np.concatenate([f32("cls_token")[None], reg]) + self.pos[: 1 + R]
        self.blocks = []
        for i in range(self.L):
            p = f"blocks.{i}."
            vecs = ("norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "attn.qkv.bias", "attn.proj.bias", "mlp.fc1.bias",
                    "mlp.fc2.bias") + (("ls1.gamma", "ls2.gamma") if vf.layer_scale else ())
            blk = {k: f32(p + k) for k in vecs}
            for k in ("attn.qkv.weight", "attn.proj.weight", "mlp.fc1.weight", "mlp.fc2.weight"):
                w = np.asarray(t[p + k], np.float32).astype(np.float16)
                if fp8 and k in ("attn.qkv.weight", "mlp.fc1.weight"):
                    q, sc = quantize_tensor(w)
                    blk[k] = (e4m3_value(q), sc)
                else:
                    blk[k] = w.astype(np.float32)
            self.blocks.append(blk)
        self.norm_w, self.norm_b = f32("norm.weight"), f32("norm.bias")
        self.w_head, self.b_head = w16("head.weight"), f32("head.bias")
        if self.pool == "map":
            lat = np.asarray(t["attn_pool.latent"], np.float64).reshape(D)
            self.q = (np.asarray(t["attn_pool.q.weight"], np.float64) @ lat + np.asarray(t["attn_pool.q.bias"], np.float64)).astype(np.float32)
            self.w_kv, self.b_kv = w16("attn_pool.kv.weight"), f32("attn_pool.kv.bias")
            self.w_pp, self.b_pp = w16("attn_pool.proj.weight"), f32("attn_pool.proj.bias")
            self.pn_w, self.pn_b = f32("attn_pool.norm.weight"), f32("attn_pool.norm.bias")
            self.w_f1, self.b_f1 = w16("attn_pool.mlp.fc1.weight"), f32("attn_pool.mlp.fc1.bias")
            self.w_f2, self.b_f2 = w16("attn_pool.mlp.fc2.weight"), f32("attn_pool.mlp.fc2.bias")

    def _mm(self, a, w):
        return (a.astype(self.acc) @ w.astype(self.acc).T).astype(np.float32)

    def _ln_linear(self, y, w):
        """qkv or fc1 on a LayerNorm's output y, without the bias: e4m3 operands in the FP8 form, f16 in the f16 form."""
        if not self.fp8:
            return self._mm(_f16(y), w)
        qw, sw = w
        qa, sa = quantize_rows(y)
        return self._mm(e4m3_value(qa), qw) * (sa * sw)[:, None]

    def _act(self, h):
        """The fc1 epilogue's activation, f16-valued."""
        with np.errstate(over="ignore"):
            return _f16(ACTIVATIONS[self.activation](np.asarray(h, np.float64)))

    def encode(self, imgs, layers=None) -> np.ndarray:
        """imgs float32 [B][S][S][C] (or [B][S][S] for one channel) -> the residual stream [B][N][D] after `layers` blocks (None: all; 0:
        the input of block 0, after the pre-norm if the model has one), as vitb200_features returns it: rows [cls, registers, patches]."""
        imgs = np.asarray(imgs, np.float32).reshape(-1, self.S, self.S, self.C)
        B, P, G, D, eps = imgs.shape[0], self.P, self.S // self.P, self.D, self.eps
        n0 = len(self.prefix)
        N = n0 + G * G
        # im2col, k = c*P*P + ky*P + kx, rounded to f16
        a = imgs.reshape(B, G, P, G, P, self.C).transpose(0, 1, 3, 5, 2, 4).reshape(B * G * G, -1)
        emb = (self._mm(_f16(a), self.w_patch) + self.b_patch).reshape(B, G * G, D) + self.pos[n0:]
        x = np.concatenate([np.broadcast_to(self.prefix, (B, n0, D)), emb], axis=1).reshape(B * N, D).astype(np.float32)
        if self.pre_norm is not None:
            x = rs.layernorm(x, *self.pre_norm, eps)
        for blk in self.blocks[:layers]:
            y = rs.layernorm(x, blk["norm1.weight"], blk["norm1.bias"], eps)
            qkv = self._ln_linear(y, blk["attn.qkv.weight"]) + blk["attn.qkv.bias"]
            qkv = qkv.reshape(B, N, 3, self.H, 64).transpose(2, 0, 3, 1, 4)  # [3][B][H][N][64]
            s = np.einsum("bhqd,bhkd->bhqk", qkv[0].astype(self.acc), qkv[1].astype(self.acc)).astype(np.float32) * np.float32(0.125)
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

    def final_ln(self, x) -> np.ndarray:
        """The final LayerNorm of every row of the residual stream [B][N][D], f32."""
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
        """The residual stream [B][N][D] -> the head's input, f32: [B * head_tokens][D] (token), [B][2 D] (cls_patch_mean) or [B][D]
        (map, mean), through the final LayerNorm first when `norm` (which the map head needs)."""
        x = np.asarray(x, np.float32)
        if self.pool == "token":
            pooled = x[:, : self.TH].reshape(-1, self.D)
            return rs.layernorm(pooled, self.norm_w, self.norm_b, self.eps) if norm else pooled
        y = self.final_ln(x) if norm else x
        if self.pool == "cls_patch_mean":
            return np.concatenate([y[:, 0], y[:, 1 + self.R:].astype(np.float64).mean(axis=1).astype(np.float32)], axis=1)
        if self.pool == "map":
            assert norm, "the attention-pooling head reads the final LayerNorm's rows"
            return self.map_head(y)
        return y.astype(np.float64).mean(axis=1).astype(np.float32)

    def forward(self, imgs) -> np.ndarray:
        """imgs float32 [B][S][S][C] -> logits [B][num_classes] ([B][head_tokens][num_classes] for more than one head token)."""
        x = self.encode(imgs)
        logits = self._mm(_f16(self.prelogits(x)), self.w_head) + self.b_head
        return logits.reshape(x.shape[0], -1) if self.TH == 1 else logits.reshape(x.shape[0], self.TH, -1)
