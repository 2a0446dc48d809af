"""Host-side mirror of the reference's vit.h interface on top of the C ABI (include/vitb200.h).

Names and argument meaning follow the reference (vit.h:118-122) so tests read like reference usage:

    model = vit_model_load(path)                      # reference vit.cpp:308  (here: parse + upload to the GPU)
    probs, idx, val = vit_predict(model, images)      # reference vit.cpp:1004 (here: batched, on the GPU)

There is NO CPU fallback: if libvitb200.so is missing or no H100 (sm_90) is present these functions raise.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import Optional

import numpy as np

from .ggml_file import ARCH_ACTIVATIONS, PATCH_ONLY_POOLS, POOLS  # vitb200_arch.activation / .pool -> name (GGUF vit.activation / vit.pool)
from .ggml_file import IMAGE_PROC_FIELDS, TEXT_POOLS, image_proc_from_config

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvitb200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "vitb200.h")
_lib = None


class VitB200Error(RuntimeError):
    pass


class Hparams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("hidden_size", "num_hidden_layers", "num_attention_heads", "num_classes",
                                          "patch_size", "img_size", "ftype")] + [("eps", C.c_float)]


class Arch(C.Structure):
    """vitb200_arch (include/vitb200.h): pre_norm 0 / 1, activation an index into ggml_file.ARCH_ACTIVATIONS, layer_scale 0 / 1,
    reg_tokens 0..16, pool an index into ggml_file.POOLS (2 and 3: SigLIP, no class token).  Fields not given are 0: Arch(pre_norm,
    activation) is a CLIP tower."""
    _fields_ = [("pre_norm", C.c_int32), ("activation", C.c_int32), ("layer_scale", C.c_int32), ("reg_tokens", C.c_int32),
                ("pool", C.c_int32)]


class ImageProc(C.Structure):
    """vitb200_image_proc (include/vitb200.h): Hugging Face's image preprocessing for the u8 entry points."""
    _fields_ = [(n, C.c_int32) for n in IMAGE_PROC_FIELDS[:6]] + [("rescale_factor", C.c_double), ("mean", C.c_float * 3),
                                                                   ("std", C.c_float * 3)]


class TextArch(C.Structure):
    """vitb200_text_arch (include/vitb200.h): a CLIP or SigLIP text tower.  pool is an index into ggml_file.TEXT_POOLS, activation one
    into ggml_file.ARCH_ACTIVATIONS; logit_scale / logit_bias are NaN when absent."""
    _fields_ = [(n, C.c_int32) for n in ("context", "causal", "pool", "eos_token_id", "activation")] + [
        ("logit_scale", C.c_float), ("logit_bias", C.c_float)]


class ZeroShot(C.Structure):
    """vitb200_zero_shot (include/vitb200.h): a zero-shot head over class embeddings [n_classes][E]."""
    _fields_ = [("class_embeds", C.c_void_p), ("n_classes", C.c_int32), ("logit_scale", C.c_float), ("logit_bias", C.c_float),
                ("mode", C.c_int32)]


ZERO_SHOT_MODES = ("softmax", "sigmoid")  # vitb200_zero_shot.mode: CLIP, SigLIP


class Taps(C.Structure):
    _fields_ = [("layer", C.c_int32)] + [(n, C.c_void_p) for n in
                                         ("embed", "ln1", "qkv", "attn", "x1", "ln2", "h", "x2", "final_ln", "x_final")]


class FeaturesReq(C.Structure):
    """vitb200_features_req (include/vitb200.h)."""
    _fields_ = [("layers", C.c_int32), ("norm", C.c_int32), ("dtype", C.c_int32)]


class Tensor(C.Structure):
    """vitb200_tensor (include/vitb200.h): one host tensor as found in vit_model::tensors (reference vit.h:88)."""
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("type", C.c_int32), ("n_dims", C.c_int32), ("ne", C.c_int64 * 4)]


def declared_symbols() -> list:
    """Every function name include/vitb200.h declares (for the CPU-side ABI test)."""
    src = open(HEADER_PATH).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vitb200_[a-z_0-9]+)\s*\(", src)))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VitB200Error(f"{LIB_PATH} is missing: build it with ./build.sh (python -c 'import __graft_entry__ as g; "
                               "g.build()'). The vit.cpp_b200 forward path has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        vp, i32, f32p = C.c_void_p, C.c_int, C.c_void_p
        L.vitb200_last_error.restype = C.c_char_p
        L.vitb200_create_from_file.argtypes = [C.c_char_p, i32, i32, C.POINTER(vp)]
        L.vitb200_create_from_file_ex.argtypes = [C.c_char_p, i32, i32, i32, C.POINTER(vp)]
        L.vitb200_create_ex.argtypes = [vp, vp, i32, i32, i32, i32, C.POINTER(vp)]
        L.vitb200_in_chans.argtypes = [vp]
        L.vitb200_head_tokens.argtypes = [vp]
        L.vitb200_create.argtypes = [vp, vp, i32, i32, i32, C.POINTER(vp)]
        L.vitb200_create_fp8.argtypes = [vp, vp, i32, i32, i32, i32, C.POINTER(vp)]
        L.vitb200_create_from_file_fp8.argtypes = [C.c_char_p, i32, i32, i32, C.POINTER(vp)]
        L.vitb200_fp8.argtypes = [vp]
        L.vitb200_mlp_dim.argtypes = [vp]
        L.vitb200_create_arch.argtypes = [vp, C.POINTER(Arch), vp, i32, i32, i32, i32, i32, C.POINTER(vp)]
        L.vitb200_get_arch.argtypes = [vp, C.POINTER(Arch)]
        L.vitb200_create_text.argtypes = [vp, C.POINTER(TextArch), vp, i32, i32, i32, i32, C.POINTER(vp)]
        L.vitb200_get_text_arch.argtypes = [vp, C.POINTER(TextArch)]
        L.vitb200_encode_text.argtypes = [vp, vp, i32, vp, C.POINTER(FeaturesReq), vp]
        L.vitb200_encode_text_device.argtypes = [vp, vp, i32, vp, C.POINTER(FeaturesReq), vp, vp]
        L.vitb200_test_attention_hilo_causal.argtypes = [i32, i32, i32, i32, vp, vp, vp]
        L.vitb200_set_image_proc.argtypes = [vp, C.POINTER(ImageProc)]
        L.vitb200_get_image_proc.argtypes = [vp, C.POINTER(ImageProc)]
        L.vitb200_set_zero_shot.argtypes = [vp, C.POINTER(ZeroShot)]
        L.vitb200_get_zero_shot.argtypes = [vp, vp, vp, vp, vp]
        L.vitb200_num_outputs.argtypes = [vp]
        L.vitb200_test_zero_shot.argtypes = [i32, i32, i32, i32, vp, vp, C.c_float, C.c_float, i32, i32, vp, vp, vp, vp]
        L.vitb200_test_quantize_fp8.argtypes = [vp, C.c_int64, vp, vp]
        L.vitb200_test_gemm_fp8.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, C.c_float, vp, vp]
        L.vitb200_test_gemm_planes.argtypes = [i32, i32, i32, i32, i32, C.c_int64, i32, vp, vp, vp, C.c_float, vp, vp, vp]
        L.vitb200_test_layernorm_fp8.argtypes = [i32, i32, i32, vp, vp, vp, C.c_float, vp, vp]
        L.vitb200_destroy.argtypes = [vp]
        L.vitb200_destroy.restype = None
        L.vitb200_get_hparams.argtypes = [vp, C.POINTER(Hparams)]
        L.vitb200_label.argtypes = [vp, i32]
        L.vitb200_label.restype = C.c_char_p
        L.vitb200_forward.argtypes = [vp, f32p, i32, f32p, f32p, vp, f32p, i32]
        L.vitb200_forward_async.argtypes = [vp, f32p, i32, f32p, f32p, vp, f32p, i32]
        L.vitb200_sync.argtypes = [vp]
        L.vitb200_profile_enable.argtypes = [vp, i32]
        L.vitb200_profile_read.argtypes = [vp, i32, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_double)]
        L.vitb200_forward_sharded.argtypes = [vp, i32, f32p, i32, f32p, f32p, vp, f32p, i32]
        L.vitb200_forward_u8.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, i32]
        L.vitb200_forward_u8_async.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, i32]
        L.vitb200_forward_device.argtypes = [vp, vp, i32, vp, vp, vp, vp, i32, vp]
        L.vitb200_recognize_u8.argtypes = [vp, vp, vp, vp, i32, vp, vp, vp, vp, vp]
        L.vitb200_recognize_u8_async.argtypes = [vp, vp, vp, vp, i32, vp, vp, vp, vp]
        L.vitb200_features.argtypes = [vp, vp, i32, C.POINTER(FeaturesReq), vp, vp]
        L.vitb200_features_device.argtypes = [vp, vp, i32, C.POINTER(FeaturesReq), vp, vp, vp]
        L.vitb200_features_u8.argtypes = [vp, vp, vp, vp, i32, i32, C.POINTER(FeaturesReq), vp, vp]
        L.vitb200_last_launch_count.argtypes = [vp]
        L.vitb200_stream.argtypes = [vp]
        L.vitb200_stream.restype = vp
        L.vitb200_forward_debug.argtypes = [vp, f32p, i32, f32p, f32p, C.POINTER(Taps)]
        L.vitb200_test_gemm.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp]
        L.vitb200_test_gemm_layer_scale.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
        L.vitb200_test_dequant.argtypes = [i32, vp, C.c_int64, vp]
        L.vitb200_test_gemm_q8.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, i32, vp]
        L.vitb200_test_layernorm.argtypes = [i32, i32, i32, vp, vp, vp, C.c_float, vp]
        L.vitb200_test_attention.argtypes = [i32, i32, i32, i32, i32, vp, vp]
        L.vitb200_test_attention_hilo.argtypes = [i32, i32, i32, i32, vp, vp, vp]
        L.vitb200_test_softmax_topk.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp]
        L.vitb200_test_attention_pool.argtypes = [i32, i32, i32, i32, vp, vp, vp]
        L.vitb200_test_attention_hd.argtypes = [i32, i32, i32, i32, i32, i32, vp, vp, vp]
        L.vitb200_test_attention_hd72.argtypes = [i32, i32, i32, i32, vp, vp, vp]
        L.vitb200_test_attention_phases.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp]
        L.vitb200_test_attention_pool_hd72.argtypes = [i32, i32, i32, i32, vp, vp, vp]
        _lib = L
    return _lib


def _check(rc: int, what: str):
    if rc != 0:
        raise VitB200Error(f"{what}: {lib().vitb200_last_error().decode()}")


class VitModel:
    """vit_model + vit_state of the reference (vit.h:72-89), living on one GPU."""

    def __init__(self, handle, device: int, max_batch: int):
        self._h = handle
        self.device = device
        self.max_batch = max_batch
        hp = Hparams()
        _check(lib().vitb200_get_hparams(self._h, C.byref(hp)), "vitb200_get_hparams")
        self.hparams = hp
        self.hidden_size, self.num_classes, self.img_size = hp.hidden_size, hp.num_classes, hp.img_size
        self.in_chans = lib().vitb200_in_chans(self._h)        # 3, or 1 for a ViTSTR model (vitstr.cpp:713); 0 for a text tower
        self.head_tokens = lib().vitb200_head_tokens(self._h)  # classifier rows per image (1, or 25 for ViTSTR)
        self.fp8 = bool(lib().vitb200_fp8(self._h))            # qkv and fc1 on the e4m3 tensor cores (vitb200_create_fp8)
        self.mlp_dim = lib().vitb200_mlp_dim(self._h)          # the MLP's hidden width: 4 D, or F read from the weights
        self._labels = None
        self._zero_shot_labels = None
        ta = TextArch()
        # a text tower (vitb200_create_text): text_arch as a dict of ggml_file.TEXT_FIELDS plus its activation; None for an image tower
        self.text_arch = None
        if self.in_chans == 0:
            _check(lib().vitb200_get_text_arch(self._h, C.byref(ta)), "vitb200_get_text_arch")
            nan = lambda x: None if x != x else float(x)
            self.text_arch = {"context": ta.context, "causal": ta.causal, "pool": TEXT_POOLS[ta.pool], "eos_token_id": ta.eos_token_id,
                              "activation": ARCH_ACTIVATIONS[ta.activation], "logit_scale": nan(ta.logit_scale), "logit_bias": nan(ta.logit_bias)}
            self.n_tokens, self.embed_dim = ta.context, hp.num_classes
            return
        self.n_tokens = (hp.img_size // hp.patch_size) ** 2 + 1
        a = Arch()
        _check(lib().vitb200_get_arch(self._h, C.byref(a)), "vitb200_get_arch")
        # the architecture (vitb200_arch): {"pre_norm": bool, "activation": one of ARCH_ACTIVATIONS}; the reference's is (False, "gelu_tanh")
        self.arch = {"pre_norm": bool(a.pre_norm), "activation": ARCH_ACTIVATIONS[a.activation]}
        # DINOv2 (vitb200_arch): LayerScale on, register tokens (rows 1 .. reg_tokens of every image), the head's input (one of POOLS)
        self.layer_scale, self.reg_tokens, self.pool = bool(a.layer_scale), int(a.reg_tokens), POOLS[a.pool]
        self.n_tokens += self.reg_tokens
        if self.pool in PATCH_ONLY_POOLS:  # SigLIP: the token rows are the patch rows only
            self.n_tokens -= 1

    @property
    def image_proc(self) -> Optional[dict]:
        """The image processor the u8 entry points use (vitb200_get_image_proc), as a dict of ggml_file.IMAGE_PROC_FIELDS; None for
        vit.cpp's preprocessing."""
        p = ImageProc()
        _check(lib().vitb200_get_image_proc(self._h, C.byref(p)), "vitb200_get_image_proc")
        if p.resample == 0:
            return None
        d = {n: getattr(p, n) for n in IMAGE_PROC_FIELDS[:7]}
        d["mean"], d["std"] = list(p.mean), list(p.std)
        return d

    def set_image_proc(self, config: Optional[dict]):
        """Give the u8 entry points Hugging Face's preprocessing (vitb200_set_image_proc): `config` is a preprocessor_config.json dict
        (ggml_file.image_proc_from_config) or a dict like image_proc returns; None restores vit.cpp's preprocessing."""
        if config is None:
            _check(lib().vitb200_set_image_proc(self._h, None), "vitb200_set_image_proc")
            return
        d = image_proc_from_config(config, self.img_size)
        p = ImageProc(*[int(d[n]) for n in IMAGE_PROC_FIELDS[:6]], float(d["rescale_factor"]), (C.c_float * 3)(*d["mean"]),
                      (C.c_float * 3)(*d["std"]))
        _check(lib().vitb200_set_image_proc(self._h, C.byref(p)), "vitb200_set_image_proc")

    @property
    def n_outputs(self) -> int:
        """Per-row width of probs and logits (vitb200_num_outputs): the zero-shot head's class count while one is set, else num_classes."""
        return lib().vitb200_num_outputs(self._h)

    @property
    def zero_shot(self) -> Optional[dict]:
        """The zero-shot head as set (vitb200_get_zero_shot): {"n_classes", "logit_scale", "logit_bias" (None for none), "probs"}; None when
        no head is set."""
        n, sc, b, mode = C.c_int32(), C.c_float(), C.c_float(), C.c_int32()
        _check(lib().vitb200_get_zero_shot(self._h, C.byref(n), C.byref(sc), C.byref(b), C.byref(mode)), "vitb200_get_zero_shot")
        if n.value == 0:
            return None
        return {"n_classes": n.value, "logit_scale": sc.value, "logit_bias": None if b.value != b.value else b.value,
                "probs": ZERO_SHOT_MODES[mode.value]}

    def set_zero_shot(self, class_embeds, logit_scale: Optional[float] = None, logit_bias: Optional[float] = None, probs: str = "softmax",
                      labels=None):
        """Classify against class embeddings on the GPU (vitb200_set_zero_shot): class_embeds [C, E] (E = num_classes, the projection
        width), usually vit_encode_text's embeds or the mean of several prompt templates per class, normalised by the engine.  Every
        prediction call then returns HF's logits_per_image over the C classes, exp(logit_scale) * cos + logit_bias, with probs "softmax"
        (CLIP) or "sigmoid" (SigLIP); logit_scale / logit_bias as the text tower stores them (text_arch).  labels: C class names that
        labels() returns while the head is set.  class_embeds None clears the head."""
        if class_embeds is None:
            _check(lib().vitb200_set_zero_shot(self._h, None), "vitb200_set_zero_shot")
            self._zero_shot_labels = None
            return
        if probs not in ZERO_SHOT_MODES:
            raise ValueError(f"probs must be one of {ZERO_SHOT_MODES}, not {probs!r}")
        if logit_scale is None:
            raise ValueError("logit_scale is required with class_embeds")
        T = np.ascontiguousarray(class_embeds, np.float32)
        if T.ndim != 2 or T.shape[1] != self.num_classes:
            raise ValueError(f"class_embeds must be [classes, {self.num_classes}], not {list(T.shape)}")
        if labels is not None and len(labels) != T.shape[0]:
            raise ValueError(f"{len(labels)} labels for {T.shape[0]} classes")
        z = ZeroShot(T.ctypes.data, T.shape[0], float(logit_scale), float("nan") if logit_bias is None else float(logit_bias),
                     ZERO_SHOT_MODES.index(probs))
        _check(lib().vitb200_set_zero_shot(self._h, C.byref(z)), "vitb200_set_zero_shot")
        self._zero_shot_labels = None if labels is None else [str(x) for x in labels]

    def label(self, i: int) -> Optional[str]:
        s = lib().vitb200_label(self._h, i)
        return s.decode() if s else None

    def labels(self) -> Optional[list]:
        """id2label as a list indexed by class id; None unless the model file names every class.  While a zero-shot head is set: the
        labels given to set_zero_shot (None if none were)."""
        if self.in_chans and self.zero_shot is not None:
            return self._zero_shot_labels
        if self._labels is None:
            self._labels = [self.label(i) for i in range(self.num_classes)]
        return None if any(s is None for s in self._labels) else self._labels

    @property
    def handle(self):
        return self._h

    def last_launch_count(self) -> int:
        return lib().vitb200_last_launch_count(self._h)

    def close(self):
        if self._h:
            lib().vitb200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def vit_model_load(fname: str, device: int = 0, max_batch: int = 256, head_tokens: int = 1, fp8: bool = False) -> VitModel:
    """reference: bool vit_model_load(const std::string &fname, vit_model &model)  (vit.cpp:308).  head_tokens = 25 loads a
    ViTSTR model (reference extensions/vitstr.cpp: 1-channel input, classifier over the first 25 tokens).  fp8 = True builds the
    FP8 engine (vitb200_create_from_file_fp8: qkv and fc1 on the e4m3 tensor cores, numerics in include/vitb200.h)."""
    h = C.c_void_p()
    create = lib().vitb200_create_from_file_fp8 if fp8 else lib().vitb200_create_from_file_ex
    _check(create(fname.encode(), device, max_batch, head_tokens, C.byref(h)), "vit_model_load")
    return VitModel(h, device, max_batch)


def vit_model_from_tensors(vf, device: int = 0, max_batch: int = 8, head_tokens: int = 1, edit=None, fp8: bool = False,
                           image_proc: Optional[dict] = None) -> VitModel:
    """vitb200_create_arch with a caller-built tensor list -- what the vit.h-side shim does with vit_model::tensors.  `vf` is a parsed
    model file (ggml_file.VitFile: numpy-shaped f32 / f16 arrays, its eps, pre_norm and activation); `edit(entries)` may reorder /
    duplicate / reshape the list of [name, array, ggml_type, ne] entries first (tests of the loader's shape and name checks).
    fp8 = True: the FP8 engine (vitb200_create_fp8).  A reference-architecture file gives what vitb200_create_ex gives.  image_proc: a
    preprocessor_config.json dict (VitModel.set_image_proc); default: the file's own (vf.image_proc), if any."""
    entries = []
    for name, arr in vf.tensors.items():
        if name.endswith(".q8_0_raw"):
            continue
        ft = vf.tensor_ftype[name]
        if ft not in (0, 1):
            raise VitB200Error("vit_model_from_tensors: f32 / f16 tensors only")
        a = np.ascontiguousarray(arr, np.float16 if ft == 1 else np.float32)
        if name == "patch_embed.proj.bias":
            a = a.reshape(1, a.size, 1, 1)  # convert-pth-to-ggml.py:150-151
        entries.append([name, a, ft, list(reversed(a.shape))])
    if edit is not None:
        entries = edit(entries) or entries
    ts = (Tensor * len(entries))()
    keep = []
    for t, (name, a, ft, ne) in zip(ts, entries):
        nm = name.encode()
        keep.append((nm, a))
        t.name, t.data, t.type, t.n_dims = nm, a.ctypes.data, ft, len(ne)
        for i in range(4):
            t.ne[i] = ne[i] if i < len(ne) else 1
    hp = Hparams(vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.num_classes, vf.patch_size, vf.img_size, vf.ftype, vf.eps)
    act = ARCH_ACTIVATIONS.index(vf.activation) if vf.activation in ARCH_ACTIVATIONS else -1  # an unknown name is refused by the engine
    h = C.c_void_p()
    if vf.text is not None:  # a text tower: vitb200_create_text
        t = vf.text
        nan = lambda x: float("nan") if x is None else float(x)
        ta = TextArch(int(t["context"]), int(t["causal"]), TEXT_POOLS.index(t["pool"]) if t["pool"] in TEXT_POOLS else -1,
                      int(t["eos_token_id"]), act, nan(t.get("logit_scale")), nan(t.get("logit_bias")))
        _check(lib().vitb200_create_text(C.byref(hp), C.byref(ta), ts, len(entries), device, max_batch, int(fp8), C.byref(h)),
               "vitb200_create_text")
        return VitModel(h, device, max_batch)
    pool = POOLS.index(vf.pool) if vf.pool in POOLS else -1  # likewise
    arch = Arch(int(vf.pre_norm), act, int(vf.layer_scale), int(vf.reg_tokens), pool)
    _check(lib().vitb200_create_arch(C.byref(hp), C.byref(arch), ts, len(entries), device, max_batch, head_tokens, int(fp8), C.byref(h)),
           "vitb200_create")
    model = VitModel(h, device, max_batch)
    image_proc = image_proc if image_proc is not None else getattr(vf, "image_proc", None)
    if image_proc is not None:
        model.set_image_proc(image_proc)
    return model


def vit_predict(model: VitModel, images: np.ndarray, topk: int = 5, want_logits: bool = False):
    """Batched reference vit_predict (vit.cpp:1004): images float32[B,S,S,3] (image_f32 layout) on the HOST.
    Returns (probs[B,C], topk_idx[B,k], topk_prob[B,k]) (+ logits[B,C] if want_logits).  For a ViTSTR model (head_tokens = n,
    images float32[B,S,S] or [B,S,S,1]) every output gains a token axis: probs[B,n,C], topk[B,n,k]."""
    imgs = np.ascontiguousarray(images, dtype=np.float32)
    ch = model.in_chans
    if imgs.ndim == (3 if ch == 3 else 2):
        imgs = imgs[None]
    B = imgs.shape[0]
    assert imgs.size == B * model.img_size * model.img_size * ch, imgs.shape
    lead = (B,) if model.head_tokens == 1 else (B, model.head_tokens)
    probs = np.empty(lead + (model.n_outputs,), np.float32)
    logits = np.empty(lead + (model.n_outputs,), np.float32) if want_logits else None
    idx = np.empty(lead + (topk,), np.int32)
    val = np.empty(lead + (topk,), np.float32)
    _check(lib().vitb200_forward(model.handle, imgs.ctypes.data, B, probs.ctypes.data,
                                 logits.ctypes.data if want_logits else None, idx.ctypes.data, val.ctypes.data, topk),
           "vit_predict")
    return (probs, idx, val, logits) if want_logits else (probs, idx, val)


def vit_predict_sharded(models, images: np.ndarray, topk: int = 5):
    """Data-parallel batched vit_predict over several VitModel engines (one per GPU) from one host thread.  Output shapes follow
    vit_predict: a ViTSTR model (head_tokens = n) returns probs[B,n,C], topk[B,n,k]; all engines must hold the same model."""
    imgs = np.ascontiguousarray(images, dtype=np.float32)
    B = imgs.shape[0]
    nc, ht = models[0].n_outputs, models[0].head_tokens
    if any(m.head_tokens != ht or m.n_outputs != nc or m.in_chans != models[0].in_chans for m in models):
        raise VitB200Error("vit_predict_sharded: the engines hold different models")
    assert imgs.size == B * models[0].img_size * models[0].img_size * models[0].in_chans, imgs.shape
    lead = (B,) if ht == 1 else (B, ht)
    probs = np.empty(lead + (nc,), np.float32)
    idx = np.empty(lead + (topk,), np.int32)
    val = np.empty(lead + (topk,), np.float32)
    hs = (C.c_void_p * len(models))(*[m.handle for m in models])
    _check(lib().vitb200_forward_sharded(hs, len(models), imgs.ctypes.data, B, probs.ctypes.data, None, idx.ctypes.data,
                                         val.ctypes.data, topk), "vit_predict_sharded")
    return probs, idx, val


def vit_predict_sharded_async(models, images: np.ndarray, probs: np.ndarray, idx: np.ndarray, val: np.ndarray):
    """Pipelined vit_predict_sharded (vitb200_forward_sharded_async): enqueues the global batch over the engines and returns; the
    caller-owned `images` / output arrays (C-contiguous, shapes as vit_predict_sharded returns them) must stay alive and untouched
    until sync_all(models).  Lets one host thread keep several global batches in flight (two pipeline slots per engine)."""
    B = images.shape[0]
    if images.dtype != np.float32 or not images.flags.c_contiguous:
        raise ValueError("images must be a C-contiguous float32 array")
    for a, dt in ((probs, np.float32), (idx, np.int32), (val, np.float32)):
        if a.dtype != dt or not a.flags.c_contiguous or a.shape[0] != B:
            raise ValueError("output arrays must be C-contiguous, one leading row per image")
    hs = (C.c_void_p * len(models))(*[m.handle for m in models])
    L = lib()
    L.vitb200_forward_sharded_async.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    _check(L.vitb200_forward_sharded_async(hs, len(models), images.ctypes.data, B, probs.ctypes.data, None, idx.ctypes.data,
                                           val.ctypes.data, idx.shape[-1]), "vit_predict_sharded_async")


def sync_all(models):
    hs = (C.c_void_p * len(models))(*[m.handle for m in models])
    L = lib()
    L.vitb200_sync_all.argtypes = [C.c_void_p, C.c_int]
    _check(L.vitb200_sync_all(hs, len(models)), "vitb200_sync_all")


def vit_image_preprocess_predict(model: VitModel, images_u8, bilinear: bool = False, topk: int = 5, predict: bool = True):
    """reference vit_image_preprocess (vit.cpp:289) + vit_predict on the GPU for a list of HxWx3 uint8 RGB arrays of any size, or the
    model's Hugging Face image processor when it has one (model.image_proc; then image_f32 is HF's pixel_values in HWC order).
    Returns (image_f32 batch [B,S,S,3], probs, topk_idx, topk_prob, logits); the last four are None if predict is False."""
    _, B, ptrs, nx, ny = _u8_batch(images_u8)
    S = model.img_size
    f32 = np.empty((B, S, S, 3), np.float32)
    probs = np.empty((B, model.n_outputs), np.float32) if predict else None
    logits = np.empty((B, model.n_outputs), np.float32) if predict else None
    idx = np.empty((B, topk), np.int32) if predict else None
    val = np.empty((B, topk), np.float32) if predict else None
    _check(lib().vitb200_forward_u8(model.handle, ptrs, nx, ny, B, int(bilinear), f32.ctypes.data,
                                    probs.ctypes.data if predict else None, logits.ctypes.data if predict else None,
                                    idx.ctypes.data if predict else None, val.ctypes.data if predict else None, topk if predict else 0),
           "vit_image_preprocess")
    return f32, probs, idx, val, logits


def _u8_batch(images_u8):
    """HxWx3 uint8 arrays -> (the contiguous arrays, which the caller keeps alive during the call, B, pointer / width / height arrays)."""
    imgs =[np.ascontiguousarray(a, dtype=np.uint8) for a in images_u8]
    B = len(imgs)
    ptrs = (C.c_void_p * B)(*[a.ctypes.data for a in imgs])
    nx = (C.c_int * B)(*[a.shape[1] for a in imgs])
    ny = (C.c_int * B)(*[a.shape[0] for a in imgs])
    return imgs, B, ptrs, nx, ny


def vitstr_recognize_u8(model: VitModel, images_u8, probs: bool = False):
    """Text recognition with a ViTSTR model (vitb200_recognize_u8): HxWx3 uint8 RGB arrays of any size >= 2x2 go through the extension's
    grayscale preprocess, the forward pass and its greedy decode (reference extensions/vitstr.cpp:128-201, 1020-1054) on the GPU.
    Returns (texts, scores float64[B], chars int32[B, n-1], lengths int32[B]) (+ probs float32[B, n, classes] if `probs`), n =
    head_tokens.  texts[b] joins model.label(id) over the decoded ids, as the extension prints them; None if the model has no id2label."""
    _, B, ptrs, nx, ny = _u8_batch(images_u8)
    n = model.head_tokens
    chars = np.empty((B, max(n - 1, 0)), np.int32)
    lengths = np.empty(B, np.int32)
    scores = np.empty(B, np.float64)
    pr = np.empty((B, n, model.num_classes), np.float32) if probs else None
    _check(lib().vitb200_recognize_u8(model.handle, ptrs, nx, ny, B, None, chars.ctypes.data, lengths.ctypes.data, scores.ctypes.data,
                                      pr.ctypes.data if probs else None), "vitstr_recognize_u8")
    names = model.labels()
    texts = None if names is None else ["".join(names[i] for i in chars[b, :lengths[b]]) for b in range(B)]
    return (texts, scores, chars, lengths, pr) if probs else (texts, scores, chars, lengths)


def vitstr_preprocess_u8(model: VitModel, images_u8) -> np.ndarray:
    """The ViTSTR extension's vit_image_preprocess (vitstr.cpp:128-201) on the GPU for HxWx3 uint8 RGB arrays: float32[B, S, S]."""
    _, B, ptrs, nx, ny = _u8_batch(images_u8)
    S = model.img_size
    out = np.empty((B, S, S), np.float32)
    _check(lib().vitb200_recognize_u8(model.handle, ptrs, nx, ny, B, out.ctypes.data, None, None, None, None), "vitstr_preprocess_u8")
    return out


BFLOAT16 = "bfloat16"  # numpy has no bf16: such features come back as uint16 bit patterns
_FEATURE_DTYPES = {np.dtype(np.float32): (0, np.float32), np.dtype(np.float16): (1, np.float16), BFLOAT16: (2, np.uint16)}


def _features_call(model: VitModel, B: int, layers, norm: bool, tokens: bool, prelogits: bool, dtype, call):
    key = dtype if isinstance(dtype, str) else np.dtype(dtype)
    if key not in _FEATURE_DTYPES:
        raise ValueError(f"dtype must be float32, float16 or {BFLOAT16!r}, not {dtype!r}")
    code, np_type = _FEATURE_DTYPES[key]
    req = FeaturesReq(model.hparams.num_hidden_layers if layers is None else int(layers), int(bool(norm)), code)
    tok = np.empty((B, model.n_tokens, model.hidden_size), np_type) if tokens else None
    # DINOv2's pool (model.pool == "cls_patch_mean"): one row of 2 D per image, class token || patch mean
    pre_shape = (B, 1, 2 * model.hidden_size) if model.pool == "cls_patch_mean" else (B, model.head_tokens, model.hidden_size)
    pre = np.empty(pre_shape, np_type) if prelogits else None
    call(C.byref(req), tok.ctypes.data if tok is not None else None, pre.ctypes.data if pre is not None else None)
    return tok, pre


def vit_features(model: VitModel, images: np.ndarray, layers=None, norm: bool = True, tokens: bool = True, prelogits: bool = False,
                 dtype=np.float32):
    """Encoder features of host images (vitb200_features): the residual stream after `layers` blocks (None = all of them; 0 = the
    embeddings), passed through the final LayerNorm when `norm`.  Returns (tokens [B,N,D], prelogits [B,head_tokens,D]), None for an
    output not asked for; with model.pool == "cls_patch_mean" (DINOv2) prelogits is [B,1,2D], the class token || the patch mean.  SigLIP
    (model.pool "map" or "mean"): tokens are the P patch rows (HF's last_hidden_state with norm, hidden_states[layers] without), prelogits
    [B,1,D] the attention-pooling head's output (HF's pooler_output; norm must be True) or the mean of the rows.  dtype float32, float16 or
    BFLOAT16 (returned as uint16 bit patterns).  Images as vit_predict takes them."""
    imgs = np.ascontiguousarray(images, dtype=np.float32)
    if imgs.ndim == (3 if model.in_chans == 3 else 2):
        imgs = imgs[None]
    B = imgs.shape[0]
    assert imgs.size == B * model.img_size * model.img_size * model.in_chans, imgs.shape
    return _features_call(model, B, layers, norm, tokens, prelogits, dtype, lambda req, t, p: _check(
        lib().vitb200_features(model.handle, imgs.ctypes.data, B, req, t, p), "vit_features"))


def vit_features_u8(model: VitModel, images_u8, bilinear: bool = False, layers=None, norm: bool = True, tokens: bool = True,
                    prelogits: bool = False, dtype=np.float32):
    """vit_features of HxWx3 uint8 RGB images of any size, pre-processed on the GPU like vit_image_preprocess_predict (through the
    model's image processor when it has one)."""
    _, B, ptrs, nx, ny = _u8_batch(images_u8)
    return _features_call(model, B, layers, norm, tokens, prelogits, dtype, lambda req, t, p: _check(
        lib().vitb200_features_u8(model.handle, ptrs, nx, ny, B, int(bilinear), req, t, p), "vit_features_u8"))


def _text_call(model: VitModel, B: int, layers, norm: bool, tokens: bool, embeds: bool, dtype, call):
    key = dtype if isinstance(dtype, str) else np.dtype(dtype)
    if key not in _FEATURE_DTYPES:
        raise ValueError(f"dtype must be float32, float16 or {BFLOAT16!r}, not {dtype!r}")
    code, np_type = _FEATURE_DTYPES[key]
    req = FeaturesReq(model.hparams.num_hidden_layers if layers is None else int(layers), int(bool(norm)), code)
    tok = np.empty((B, model.n_tokens, model.hidden_size), np_type) if tokens else None
    emb = np.empty((B, model.embed_dim), np.float32) if embeds else None
    call(emb.ctypes.data if emb is not None else None, C.byref(req), tok.ctypes.data if tok is not None else None)
    return emb, tok


def vit_encode_text(model: VitModel, ids, layers=None, norm: bool = True, tokens: bool = False, embeds: bool = True, dtype=np.float32):
    """A text tower on token ids (vitb200_encode_text): ids int [B, N] (or [N]) from the model's Hugging Face tokenizer, padded to the
    context length N.  Returns (embeds float32 [B, E], tokens [B, N, D]), None for an output not asked for: embeds are HF's text_embeds
    (pooler_output for CLIPTextModel); tokens the residual stream after `layers` blocks (None = all), through the final LayerNorm when
    `norm` (layers = L - 1, norm = False: hidden_states[-2]), as float32, float16 or BFLOAT16 (uint16 bit patterns).  An id outside the
    vocabulary is refused."""
    x = np.ascontiguousarray(ids, np.int32)
    if x.ndim == 1:
        x = x[None]
    if x.ndim != 2 or x.shape[1] != model.n_tokens:
        raise ValueError(f"ids must be [batch, {model.n_tokens}] (padded to the context length), not {list(x.shape)}")
    return _text_call(model, x.shape[0], layers, norm, tokens, embeds, dtype, lambda e, req, t: _check(
        lib().vitb200_encode_text(model.handle, x.ctypes.data, x.shape[0], e, req, t), "vit_encode_text"))


def zero_shot_logits(image_embeds, text_embeds, logit_scale: float, logit_bias: Optional[float] = None) -> np.ndarray:
    """Hugging Face's logits_per_image on the host: both embeddings L2-normalised, exp(logit_scale) * img @ txt.T, + logit_bias for
    SigLIP.  image_embeds [I, E], text_embeds [T, E] -> [I, T] (float64).  The float64 check of VitModel.set_zero_shot, which computes
    the same scores on the GPU."""
    img = np.asarray(image_embeds, np.float64)
    txt = np.asarray(text_embeds, np.float64)
    img = img / np.linalg.norm(img, axis=-1, keepdims=True)
    txt = txt / np.linalg.norm(txt, axis=-1, keepdims=True)
    logits = np.exp(logit_scale) * img @ txt.T
    return logits if logit_bias is None else logits + logit_bias


TAP_SHAPES = {
    "embed": lambda B, N, D: (B, N, D), "ln1": lambda B, N, D: (B, N, D), "qkv": lambda B, N, D: (B, N, 3 * D),
    "attn": lambda B, N, D: (B, N, D), "x1": lambda B, N, D: (B, N, D), "ln2": lambda B, N, D: (B, N, D),
    "h": lambda B, N, D: (B, N, 4 * D), "x2": lambda B, N, D: (B, N, D), "final_ln": lambda B, N, D: (B, D),
    "x_final": lambda B, N, D: (B, N, D),
}


def vit_predict_debug(model: VitModel, images: np.ndarray, tap_layer: int, taps=tuple(TAP_SHAPES)):
    """Forward with intermediates copied back (tests only).  For a ViTSTR model (head_tokens = n) the outputs and the final_ln tap
    gain a token axis, as in vit_predict."""
    imgs = np.ascontiguousarray(images, dtype=np.float32)
    if imgs.ndim == (3 if model.in_chans == 3 else 2):
        imgs = imgs[None]
    B = imgs.shape[0]
    lead = (B,) if model.head_tokens == 1 else (B, model.head_tokens)
    probs = np.empty(lead + (model.n_outputs,), np.float32)
    logits = np.empty(lead + (model.n_outputs,), np.float32)
    tp = Taps()
    tp.layer = tap_layer
    out = {}
    for n in taps:
        shape = TAP_SHAPES[n](B, model.n_tokens, model.hidden_size)
        if n == "final_ln" and model.pool == "cls_patch_mean":
            shape = (B, 2 * model.hidden_size)
        if n == "h":
            shape = (B, model.n_tokens, model.mlp_dim)
        out[n] = np.zeros(lead + shape[1:] if n == "final_ln" else shape, np.float32)
        setattr(tp, n, out[n].ctypes.data)
    _check(lib().vitb200_forward_debug(model.handle, imgs.ctypes.data, B, probs.ctypes.data, logits.ctypes.data,
                                       C.byref(tp)), "vit_predict_debug")
    return probs, logits, out


# attention kernels of vitb200_test_attention (include/vitb200.h): engine's choice, mma.sync with 8 warps (any N), wgmma (N <= 224,
# the split-precision kernel the engine picks for N: persistent up to 200 tokens, one CTA per (image, head) beyond), mma.sync with 16
# warps (128 < N <= 640); the head-dim-80 kernel (vitb200_test_attention_hd); the one-CTA-per-(image, head) wgmma kernel at any N <= 224
ATTN_AUTO, ATTN_MMA8, ATTN_WGMMA, ATTN_MMA16, ATTN_MMA80, ATTN_WGMMA_HEAD = 0, 1, 2, 3, 4, 5


def test_attention(qkv16: np.ndarray, B: int, N: int, H: int, kernel: int = ATTN_AUTO, device: int = 0) -> np.ndarray:
    """Stand-alone attention kernel: qkv16 float16 [B*N, 3*H*64] -> float32 [B*N, H*64]."""
    q = np.ascontiguousarray(qkv16, np.float16).reshape(B * N, 3 * H * 64)
    out = np.empty((B * N, H * 64), np.float32)
    _check(lib().vitb200_test_attention(device, kernel, B, N, H, q.ctypes.data, out.ctypes.data), "vitb200_test_attention")
    return out


def split_hi_lo(x: np.ndarray):
    """x (float32) -> (hi, lo) float16 with hi = f16(x), lo = f16(x - hi): what the qkv GEMM's split-precision epilogue stores."""
    x = np.ascontiguousarray(x, np.float32)
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def test_attention_hilo(qkv32: np.ndarray, B: int, N: int, H: int, device: int = 0) -> np.ndarray:
    """The wgmma attention kernel (N <= 224) on split-precision operands: qkv32 float32 [B*N, 3*H*64] is passed as hi + lo."""
    hi, lo = split_hi_lo(np.asarray(qkv32, np.float32).reshape(B * N, 3 * H * 64))
    out = np.empty((B * N, H * 64), np.float32)
    _check(lib().vitb200_test_attention_hilo(device, B, N, H, hi.ctypes.data, lo.ctypes.data, out.ctypes.data),
           "vitb200_test_attention_hilo")
    return out


def test_attention_hilo_causal(qkv32: np.ndarray, B: int, N: int, H: int, device: int = 0) -> np.ndarray:
    """test_attention_hilo with CLIP's causal mask (vitb200_test_attention_hilo_causal): query t attends to keys 0 .. t."""
    hi, lo = split_hi_lo(np.asarray(qkv32, np.float32).reshape(B * N, 3 * H * 64))
    out = np.empty((B * N, H * 64), np.float32)
    _check(lib().vitb200_test_attention_hilo_causal(device, B, N, H, hi.ctypes.data, lo.ctypes.data, out.ctypes.data),
           "vitb200_test_attention_hilo_causal")
    return out


def test_attention_hd(qkv32: np.ndarray, B: int, N: int, H: int, hd: int, split: bool, kernel: int = ATTN_AUTO,
                      device: int = 0) -> np.ndarray:
    """The attention kernel of head dim hd (64 or 80) alone (vitb200_test_attention_hd): qkv32 float32 [B*N, 3*H*hd], row-major
    q | k | v, passed as hi + lo (split_hi_lo) when `split`, else as its f16 values -> float32 [B*N, H*hd]."""
    x = np.ascontiguousarray(qkv32, np.float32).reshape(B * N, 3 * H * hd)
    hi, lo = split_hi_lo(x) if split else (x.astype(np.float16), None)
    out = np.empty((B * N, H * hd), np.float32)
    _check(lib().vitb200_test_attention_hd(device, kernel, B, N, H, hd, hi.ctypes.data, None if lo is None else lo.ctypes.data,
                                           out.ctypes.data), "vitb200_test_attention_hd")
    return out


# the phase probe's records: per CTA, ATTN_PROBE_PROBLEMS problems of ATTN_PROBE_FIELDS stamps (csrc/attention_wgmma.cuh)
ATTN_PROBE_PROBLEMS, ATTN_PROBE_FIELDS = 64, 9


def test_attention_phases(qkv32: np.ndarray, B: int, N: int, H: int, kernel: int = ATTN_WGMMA, device: int = 0) -> np.ndarray:
    """The split-precision wgmma kernel `kernel` (ATTN_WGMMA or ATTN_WGMMA_HEAD) with its phase probe on (vitb200_test_attention_phases):
    qkv32 float32 [B*N, 3*H*64] passed as hi + lo -> uint64 %globaltimer stamps [grid, ATTN_PROBE_PROBLEMS, ATTN_PROBE_FIELDS] in ns,
    0 where nothing was recorded."""
    hi, lo = split_hi_lo(np.asarray(qkv32, np.float32).reshape(B * N, 3 * H * 64))
    rec = np.zeros(B * H * ATTN_PROBE_PROBLEMS * ATTN_PROBE_FIELDS, np.uint64)
    grid = C.c_int(0)
    _check(lib().vitb200_test_attention_phases(device, kernel, B, N, H, hi.ctypes.data, lo.ctypes.data, rec.ctypes.data, C.byref(grid)),
           "vitb200_test_attention_phases")
    return rec[:grid.value * ATTN_PROBE_PROBLEMS * ATTN_PROBE_FIELDS].reshape(grid.value, ATTN_PROBE_PROBLEMS, ATTN_PROBE_FIELDS)


def test_attention_hd72(qkv32: np.ndarray, B: int, N: int, H: int, split: bool, device: int = 0) -> np.ndarray:
    """The head-dim-72 attention kernel alone (vitb200_test_attention_hd72), as test_attention_hd takes its operands: qkv32 float32
    [B*N, 3*H*72], row-major q | k | v, split into hi + lo when `split` (N <= 224), else its f16 values -> float32 [B*N, H*72]."""
    x = np.ascontiguousarray(qkv32, np.float32).reshape(B * N, 3 * H * 72)
    hi, lo = split_hi_lo(x) if split else (x.astype(np.float16), None)
    out = np.empty((B * N, H * 72), np.float32)
    _check(lib().vitb200_test_attention_hd72(device, B, N, H, hi.ctypes.data, None if lo is None else lo.ctypes.data, out.ctypes.data),
           "vitb200_test_attention_hd72")
    return out


def test_attention_parts(hi: np.ndarray, lo: np.ndarray, B: int, N: int, H: int, hd: int, causal: bool = False,
                         device: int = 0) -> np.ndarray:
    """The split-precision attention kernel of head dim hd (64, 80 or 72; N <= 224) on hi and lo halves passed as given: hi, lo
    float16 [B*N, 3*H*hd], row-major q | k | v -> float32 [B*N, H*hd].  Nothing requires lo to be the rounding residue of hi, so an
    operand can live in one half alone and each of S = Ql Kh^T + Qh Kl^T + Qh Kh^T and O = P Vl + P Vh be exercised by itself.
    causal (CLIP's mask) runs at head dim 64 only, where the causal kernel is."""
    if causal and hd != 64:
        raise ValueError(f"the causal mask runs at head dim 64 only, not {hd}")
    h = np.ascontiguousarray(hi, np.float16).reshape(B * N, 3 * H * hd)
    l = np.ascontiguousarray(lo, np.float16).reshape(B * N, 3 * H * hd)
    out = np.empty((B * N, H * hd), np.float32)
    L = lib()
    if hd == 64:
        name = "vitb200_test_attention_hilo_causal" if causal else "vitb200_test_attention_hilo"
        rc = getattr(L, name)(device, B, N, H, h.ctypes.data, l.ctypes.data, out.ctypes.data)
    elif hd == 80:
        name = "vitb200_test_attention_hd"
        rc = L.vitb200_test_attention_hd(device, ATTN_AUTO, B, N, H, hd, h.ctypes.data, l.ctypes.data, out.ctypes.data)
    elif hd == 72:
        name = "vitb200_test_attention_hd72"
        rc = L.vitb200_test_attention_hd72(device, B, N, H, h.ctypes.data, l.ctypes.data, out.ctypes.data)
    else:
        raise ValueError(f"split-precision attention runs head dims 64, 80 and 72, not {hd}")
    _check(rc, name)
    return out


def test_attention_pool_hd72(q: np.ndarray, kv16: np.ndarray, B: int, P: int, H: int, device: int = 0) -> np.ndarray:
    """test_attention_pool at head dim 72 (vitb200_test_attention_pool_hd72): q float32 [H*72], kv16 float16 [B*P, 2*H*72] (every row
    k then v) -> float32 [B, H*72], the f16 results of sum_j softmax_j(q_h k_j / sqrt(72)) v_j."""
    qq = np.ascontiguousarray(q, np.float32).reshape(H * 72)
    kv = np.ascontiguousarray(kv16, np.float16).reshape(B * P, 2 * H * 72)
    out = np.empty((B, H * 72), np.float32)
    _check(lib().vitb200_test_attention_pool_hd72(device, B, P, H, qq.ctypes.data, kv.ctypes.data, out.ctypes.data),
           "vitb200_test_attention_pool_hd72")
    return out


def test_attention_pool(q: np.ndarray, kv16: np.ndarray, B: int, P: int, H: int, device: int = 0) -> np.ndarray:
    """The attention-pooling head's attention kernel alone (vitb200_test_attention_pool): q float32 [H*64] (one query per head), kv16
    float16 [B*P, 2*H*64] (every row k then v) -> float32 [B, H*64], the f16 results of sum_j softmax_j(q_h k_j / 8) v_j."""
    qq = np.ascontiguousarray(q, np.float32).reshape(H * 64)
    kv = np.ascontiguousarray(kv16, np.float16).reshape(B * P, 2 * H * 64)
    out = np.empty((B, H * 64), np.float32)
    _check(lib().vitb200_test_attention_pool(device, B, P, H, qq.ctypes.data, kv.ctypes.data, out.ctypes.data), "vitb200_test_attention_pool")
    return out


def test_softmax_topk(logits: np.ndarray, k: int, device: int = 0):
    """The classifier's soft-max + top-k kernel alone (vitb200_test_softmax_topk): logits float32 [rows][C] -> (probs float32
    [rows][C], topk_idx int32 [rows][k], topk_val float32 [rows][k])."""
    x = np.ascontiguousarray(logits, np.float32)
    rows, C = x.shape
    probs = np.empty((rows, C), np.float32)
    idx = np.empty((rows, k), np.int32)
    val = np.empty((rows, k), np.float32)
    _check(lib().vitb200_test_softmax_topk(device, rows, C, k, x.ctypes.data, probs.ctypes.data, idx.ctypes.data if k else None,
                                           val.ctypes.data if k else None), "vitb200_test_softmax_topk")
    return probs, idx, val


def test_zero_shot(x, class_embeds, logit_scale: float, logit_bias: Optional[float] = None, probs: str = "softmax", k: int = 0,
                   device: int = 0):
    """The zero-shot head's kernels alone (vitb200_test_zero_shot): head rows x float32 [rows][E], raw class rows [C][E] -> (probs
    float32 [rows][C], scores float32 [rows][C], topk_idx int32 [rows][k], topk_val float32 [rows][k])."""
    X = np.ascontiguousarray(x, np.float32)
    T = np.ascontiguousarray(class_embeds, np.float32)
    rows, E = X.shape
    n = T.shape[0]
    pr = np.empty((rows, n), np.float32)
    lg = np.empty((rows, n), np.float32)
    idx = np.empty((rows, k), np.int32)
    val = np.empty((rows, k), np.float32)
    _check(lib().vitb200_test_zero_shot(device, rows, E, n, X.ctypes.data, T.ctypes.data, float(logit_scale),
                                        float("nan") if logit_bias is None else float(logit_bias), ZERO_SHOT_MODES.index(probs), k,
                                        pr.ctypes.data, lg.ctypes.data, idx.ctypes.data if k else None, val.ctypes.data if k else None),
           "vitb200_test_zero_shot")
    return pr, lg, idx, val


def test_dequant(ggml_type: int, blocks: np.ndarray) -> np.ndarray:
    """Host-only: the engine's upload-time conversion of quantised blocks -> float16[n_blocks*32]."""
    from .ggml_file import QUANT_BLOCK_BYTES
    raw = np.ascontiguousarray(blocks, np.uint8).reshape(-1)
    nb = raw.size // QUANT_BLOCK_BYTES[ggml_type]
    out = np.empty(nb * 32, np.uint16)
    _check(lib().vitb200_test_dequant(ggml_type, raw.ctypes.data, nb, out.ctypes.data), "vitb200_test_dequant")
    return out.view(np.float16)


# The GEMM epilogue ids of vitb200_test_gemm / vitb200_test_gemm_fp8, named as in enum GemmEpilogue (csrc/gemm_wgmma.cuh)
EPI_BIAS_F16 = 0
EPI_BIAS_GELU_F16 = 1
EPI_BIAS_RESID_F32 = 2
EPI_PATCH_F32 = 3
EPI_BIAS_F32 = 4
EPI_BIAS_F16_HILO = 6
EPI_BIAS_GELU_ERF_F16 = 7
EPI_BIAS_QUICK_GELU_F16 = 8
EPI_BIAS_SCALE_RESID_F32 = 9
EPI_BIAS_GELU_PYTORCH_TANH_F16 = 10
EPI_BIAS_SWIGLU_F16 = 11  # W [N][K] in HF's order (N = 2 F), out [M][N / 2]
EPI_SWIGLU = EPI_BIAS_SWIGLU_F16


def test_gemm(M: int, N: int, K: int, epilogue: int, A16: np.ndarray, W16: np.ndarray, bias: np.ndarray,
              resid: Optional[np.ndarray] = None, device: int = 0) -> np.ndarray:
    A = np.ascontiguousarray(A16, np.float16)
    W = np.ascontiguousarray(W16, np.float16)
    b = np.ascontiguousarray(bias, np.float32)
    r = np.ascontiguousarray(resid, np.float32) if resid is not None else None
    out = np.empty((M, N // 2 if epilogue == EPI_SWIGLU else N), np.float32)
    _check(lib().vitb200_test_gemm(device, M, N, K, epilogue, A.ctypes.data, W.ctypes.data, b.ctypes.data,
                                   r.ctypes.data if r is not None else None, out.ctypes.data), "vitb200_test_gemm")
    return out


def test_gemm_layer_scale(M: int, N: int, K: int, A16: np.ndarray, W16: np.ndarray, bias: np.ndarray, gamma: np.ndarray,
                          resid: np.ndarray, device: int = 0) -> np.ndarray:
    """The LayerScale residual epilogue alone (vitb200_test_gemm_layer_scale): f32(f32(A W^T + bias) * gamma) + resid, [M][N] f32."""
    A = np.ascontiguousarray(A16, np.float16)
    W = np.ascontiguousarray(W16, np.float16)
    b, g, r = (np.ascontiguousarray(x, np.float32) for x in (bias, gamma, resid))
    out = np.empty((M, N), np.float32)
    _check(lib().vitb200_test_gemm_layer_scale(device, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data, g.ctypes.data, r.ctypes.data,
                                               out.ctypes.data), "vitb200_test_gemm_layer_scale")
    return out


def test_gemm_q8(x, w_blocks, bias, device: int = 0, iters: int = 0):
    """The q8_0 linear layer on the integer tensor cores (vitb200_test_gemm_q8): x float32 [M][K], w_blocks = uint8 bytes of a q8_0
    tensor [N][K/32] blocks (model-file layout), bias [N].  Returns (y [M][N] f32, xq [M][K] int8, xd [M][K/32] f32, ms per launch or None)."""
    x = np.ascontiguousarray(x, np.float32)
    w = np.ascontiguousarray(w_blocks, np.uint8)
    b = np.ascontiguousarray(bias, np.float32)
    M, K = x.shape
    N = b.shape[0]
    if w.size != N * (K // 32) * 34:
        raise ValueError("w_blocks does not hold N * K / 32 q8_0 blocks")
    y = np.empty((M, N), np.float32)
    xq = np.empty((M, K), np.int8)
    xd = np.empty((M, K // 32), np.float32)
    ms = C.c_float(0.0)
    _check(lib().vitb200_test_gemm_q8(device, M, N, K, x.ctypes.data, w.ctypes.data, b.ctypes.data, y.ctypes.data, xq.ctypes.data,
                                      xd.ctypes.data, iters, C.cast(C.pointer(ms), C.c_void_p)), "vitb200_test_gemm_q8")
    return y, xq, xd, (ms.value if iters > 0 else None)


def test_layernorm(x, w, b, eps: float = 1e-6, device: int = 0):
    """The block LayerNorm kernel alone (vitb200_test_layernorm): x float32 [rows][D] -> float32 [rows][D] (f16 values widened)."""
    x = np.ascontiguousarray(x, np.float32)
    w = np.ascontiguousarray(w, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    y = np.empty_like(x)
    _check(lib().vitb200_test_layernorm(device, x.shape[0], x.shape[1], x.ctypes.data, w.ctypes.data, b.ctypes.data, eps, y.ctypes.data),
           "vitb200_test_layernorm")
    return y


def test_quantize_fp8(w16: np.ndarray):
    """Host-only: the FP8 engine's weight quantisation (vitb200_test_quantize_fp8): float16 array -> (uint8 e4m3 bytes, same shape;
    f32 scale)."""
    w = np.ascontiguousarray(w16, np.float16)
    q = np.empty(w.shape, np.uint8)
    sc = C.c_float(0.0)
    _check(lib().vitb200_test_quantize_fp8(w.ctypes.data, w.size, q.ctypes.data, C.cast(C.pointer(sc), C.c_void_p)),
           "vitb200_test_quantize_fp8")
    return q, sc.value


def test_gemm_fp8(M: int, N: int, K: int, epilogue: int, A8: np.ndarray, a_scale: np.ndarray, W8: np.ndarray, w_scale: float,
                  bias: np.ndarray, device: int = 0) -> np.ndarray:
    """The e4m3 GEMM alone (vitb200_test_gemm_fp8): A8 uint8 [M][K], W8 uint8 [N][K] e4m3 bytes -> float32 [M][N] ([M][N / 2] for
    EPI_SWIGLU)."""
    A = np.ascontiguousarray(A8, np.uint8)
    W = np.ascontiguousarray(W8, np.uint8)
    sa = np.ascontiguousarray(a_scale, np.float32)
    b = np.ascontiguousarray(bias, np.float32)
    out = np.empty((M, N // 2 if epilogue == EPI_SWIGLU else N), np.float32)
    _check(lib().vitb200_test_gemm_fp8(device, M, N, K, epilogue, A.ctypes.data, sa.ctypes.data, W.ctypes.data, float(w_scale),
                                       b.ctypes.data, out.ctypes.data), "vitb200_test_gemm_fp8")
    return out


def test_gemm_planes(M: int, N: int, K: int, epilogue: int, A: np.ndarray, W: np.ndarray, bias: np.ndarray, plane_rows: int,
                     a_scale: Optional[np.ndarray] = None, w_scale: float = 1.0, device: int = 0):
    """The qkv / k | v GEMM with head-major output (vitb200_test_gemm_planes): A [M][K] and W [N][K] float16, or e4m3 bytes (uint8) when
    a_scale is given -> (hi, lo) uint16 f16 bits [N // 64][plane_rows][64], lo None for EPI_BIAS_F16.  Rows past M hold 0xFFFF."""
    e4m3 = a_scale is not None
    dt = np.uint8 if e4m3 else np.float16
    A, W = np.ascontiguousarray(A, dt), np.ascontiguousarray(W, dt)
    b = np.ascontiguousarray(bias, np.float32)
    sa = np.ascontiguousarray(a_scale, np.float32) if e4m3 else None
    planes = (max(N, 0) // 64, max(plane_rows, 0), 64)
    hi = np.empty(planes, np.uint16)
    lo = np.empty(planes, np.uint16) if epilogue == EPI_BIAS_F16_HILO else None
    _check(lib().vitb200_test_gemm_planes(device, M, N, K, epilogue, plane_rows, int(e4m3), A.ctypes.data, sa.ctypes.data if e4m3 else None,
                                          W.ctypes.data, float(w_scale), b.ctypes.data, hi.ctypes.data,
                                          lo.ctypes.data if lo is not None else None), "vitb200_test_gemm_planes")
    return hi, lo


def test_layernorm_fp8(x, w, b, eps: float = 1e-6, device: int = 0):
    """The FP8 engine's block LayerNorm alone (vitb200_test_layernorm_fp8): x float32 [rows][D] -> (uint8 e4m3 [rows][D], float32 [rows])."""
    x = np.ascontiguousarray(x, np.float32)
    w = np.ascontiguousarray(w, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    q = np.empty(x.shape, np.uint8)
    sa = np.empty(x.shape[0], np.float32)
    _check(lib().vitb200_test_layernorm_fp8(device, x.shape[0], x.shape[1], x.ctypes.data, w.ctypes.data, b.ctypes.data, eps,
                                            q.ctypes.data, sa.ctypes.data), "vitb200_test_layernorm_fp8")
    return q, sa
