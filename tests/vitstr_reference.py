"""The ViTSTR extension's own preprocess and decode, as test oracles.

preprocess(): the extension's vit_image_preprocess (reference extensions/vitstr.cpp:135-201) run inside the compiled extension
(oracle/_ref/libvitstrref.so exports it).  It is a C++ function, `bool vit_image_preprocess(const image_u8&, image_f32&, const
vit_hparams&)`, so it is called with argument objects laid out as gcc/libstdc++ lays out those structs (vitstr.h:22-38, 92-104):
a std::vector<T> is three pointers {begin, end, end of storage}.  The output vector already has S*S elements, so the function's
`res.data.resize(S*S, 0)` is a no-op and it writes straight into the numpy array; of the hyper-parameters it reads img_size only
(n_img_size(), vitstr.cpp:33-36).

gray_level(): the extension's rgb_to_grayscale (vitstr.cpp:128-132) for a gray pixel (v, v, v), emulated exactly with rationals:
the build computes fma(0.114, b, fma(0.299, r, 0.587 * g)) in double and truncates.

greedy_decode(): the extension's decode loop (vitstr.cpp:1020-1054) in numpy, on a [B][n][classes] probability array."""
import ctypes as C
from fractions import Fraction

import numpy as np

from oracle import ref

_PREPROCESS = "_Z20vit_image_preprocessRK8image_u8R9image_f32RK11vit_hparams"


def available() -> bool:
    return ref.vitstr_available()


class _Vec(C.Structure):
    _fields_ = [("begin", C.c_void_p), ("end", C.c_void_p), ("cap", C.c_void_p)]


class _Image(C.Structure):
    _fields_ = [("nx", C.c_int), ("ny", C.c_int), ("data", _Vec)]


class _Hparams(C.Structure):
    # seven int32 + float eps, then std::map<int, std::string> id2label (48 bytes in libstdc++; never touched by the preprocess)
    _fields_ = [(n, C.c_int32) for n in ("hidden_size", "num_hidden_layers", "num_attention_heads", "num_classes", "patch_size",
                                          "img_size", "ftype")] + [("eps", C.c_float), ("id2label", C.c_uint8 * 64)]


def _vec(a: np.ndarray) -> _Vec:
    p = a.ctypes.data
    return _Vec(p, p + a.nbytes, p + a.nbytes)


def preprocess(rgb_u8: np.ndarray, img_size: int) -> np.ndarray:
    """The extension's vit_image_preprocess on one HxWx3 uint8 image: float32[S, S]."""
    fn = getattr(ref.vitstr_lib(), _PREPROCESS)
    fn.restype = C.c_bool
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    rgb = np.ascontiguousarray(rgb_u8, np.uint8)
    ny, nx, _ = rgb.shape
    out = np.zeros((img_size, img_size), np.float32)
    src, dst = _Image(nx, ny, _vec(rgb)), _Image(0, 0, _vec(out))
    hp = _Hparams()
    hp.img_size = img_size
    if not fn(C.byref(src), C.byref(dst), C.byref(hp)):
        raise RuntimeError("the extension's vit_image_preprocess failed")
    assert (dst.nx, dst.ny) == (img_size, img_size) and dst.data.begin == out.ctypes.data  # it wrote into `out`, no reallocation
    return out


def _round_double(q: Fraction) -> Fraction:
    return Fraction(float(q))  # int / int true division in Python is correctly rounded: float(Fraction) is round-to-nearest-even


def gray_level(v: int) -> int:
    t = _round_double(Fraction(0.587) * v)
    t = _round_double(Fraction(0.299) * v + t)
    t = _round_double(Fraction(0.114) * v + t)
    return int(t)  # truncation, as the (uint8_t) cast of a non-negative double


def greedy_decode(probs: np.ndarray):
    """probs float32 [B][n][classes] -> (chars int32 [B][n-1] (-1 past the end), lengths int32 [B], scores float64 [B])."""
    B, n, _ = probs.shape
    chars = np.full((B, n - 1), -1, np.int32)
    lengths = np.zeros(B, np.int32)
    scores = np.ones(B, np.float64)
    for b in range(B):
        conf = 1.0
        for t in range(1, n):
            i = int(np.argmax(probs[b, t]))  # first index of the maximum == the extension's `>` scan from class 0
            if i == 1:
                break
            conf *= float(probs[b, t, i])
            chars[b, t - 1] = i
            lengths[b] += 1
        scores[b] = conf
    return chars, lengths, scores
