"""The FP8 engine's quantisation (vitb200_create_fp8, numerics in include/vitb200.h) and the distance the tests measure, for tests.

qkv and fc1 run on e4m3 operands, every other GEMM stays f16 (tests/emulation.py runs the whole forward pass):

    y   = LayerNorm(x)                      f32, per token row
    sa  = amax(|y|) / 448,  qa = e4m3(y * (448 / amax))          (scale 1 for an all-zero row)
    sw  = amax(|w16|) / 448, qw = e4m3(w16 * (448 / amax))       (per tensor)
    out = sum_k qa qw * (sa * sw) + bias                         then the f16 engine's epilogue (qkv: f32; fc1: f16, GELU, f16)"""
import numpy as np
import torch

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


def rel_dist(a, b) -> np.ndarray:
    """Per image max|a - b| / max|b| over the last axis (and the token axis, if any)."""
    a = np.asarray(a, np.float64).reshape(a.shape[0], -1)
    b = np.asarray(b, np.float64).reshape(b.shape[0], -1)
    return np.abs(a - b).max(axis=1) / np.abs(b).max(axis=1)
