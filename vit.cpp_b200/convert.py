"""Offline converters for ViT checkpoints -- the timm-free counterpart of the reference's convert-pth-to-ggml.py and quantize.cpp.

    python -m convert <checkpoint.pth|.safetensors> <out.gguf> [--ftype 0|1] [--heads H] [--labels labels.json] [--container legacy|gguf]
                      [--keep-norm-pre] [--activation gelu_tanh|gelu_erf|quick_gelu] [--eps E]     (timm; these three need GGUF)
    python -m convert <CLIP model.safetensors|.pth> <out.gguf> --hf-config config.json             (Hugging Face CLIP vision tower)
    python -m convert <DINOv2 model.safetensors> <out.gguf> --hf-config config.json [--img-size S]  (Hugging Face DINOv2)
    python -m convert <SigLIP model.safetensors> <out.gguf> --hf-config config.json               (Hugging Face SigLIP vision tower)
    python -m convert <any of the above, or a converted model file> <out.gguf> ... --hf-preprocessor preprocessor_config.json
                                                                    (the u8 entry points prepare images as this HF image processor does)
    python -m convert <CLIP or SigLIP model.safetensors> <out.gguf> --hf-config config.json --text     (the text tower)
    python -m convert --quantize <in.gguf> <out.gguf> q8_0

* `state_dict_to_model_file` follows reference convert-pth-to-ggml.py:105-158 step by step (header, id2label table, tensors in
  state_dict order, `norm_pre*` skipped, 1-D tensors + pos_embed + cls_token kept f32, the conv bias reshaped to (1, D, 1, 1)),
  but takes the weights from a plain `state_dict` -- a torch checkpoint (`torch.load`, needs torch) or a .safetensors file (read
  here with numpy only) -- instead of instantiating the model through timm.  Hyper-parameters are inferred from the tensor shapes
  (timm `VisionTransformer` names, reference vit.cpp:518-579); the head count is not recoverable from shapes and defaults to
  hidden / 64 (true for every timm ViT the reference lists).
* `clip_to_model_file` converts a Hugging Face CLIP vision tower (`vision_model.*` of CLIPVisionModel, CLIPVisionModelWithProjection
  or CLIPModel) to a GGUF file with the pre-norm, QuickGELU or erf GELU and eps 1e-5 (`clip_to_timm` holds the name mapping).
* `dinov2_to_model_file` converts a Hugging Face DINOv2 (Dinov2Model, Dinov2WithRegistersModel and their ForImageClassification
  heads) to a GGUF file with LayerScale, register tokens and, with a classifier, the class-plus-patch-mean head (`dinov2_to_timm`).
  `--img-size S` resamples the patch position grid of any converted model to S / patch, as Hugging Face does at run time.
* `siglip_to_model_file` converts a Hugging Face SigLIP vision tower (SiglipVisionModel, the vision tower of SiglipModel, or
  SiglipForImageClassification) to a GGUF file without a class token, with PyTorch's tanh GELU and the attention-pooling head (pool 'map')
  or, with a classifier, the token mean (pool 'mean') (`siglip_to_timm`).
* `text_to_model_file` converts the text tower of a Hugging Face CLIP (CLIPTextModel, CLIPTextModelWithProjection, CLIPModel) or SigLIP
  (SiglipTextModel, SiglipModel) to a GGUF text file (vitb200_text_arch: token table, causal mask for CLIP, EOS or last-row pooling, the
  projection as the head, logit_scale / logit_bias as metadata) (`text_to_timm`).  Tokenisation stays with the caller's HF tokenizer.
* `quantize_model_file` restates reference quantize.cpp for q8_0 (every 2-D `*weight` tensor, quantize_row_q8_0_reference,
  ggml-quants.c): byte-identical to the reference binary's output (pinned by the CPU test-suite).

Host-side tooling: nothing here touches the GPU or the test infrastructure.
"""
from __future__ import annotations

import json
import re
import struct
import sys
from typing import Dict, Optional

import numpy as np

try:  # package import (vit_cpp_b200.convert) or plain script next to ggml_file.py
    from . import ggml_file as gf
except ImportError:  # pragma: no cover
    import ggml_file as gf

_ST_DTYPES = {"F32": np.float32, "F16": np.float16, "F64": np.float64, "I64": np.int64, "I32": np.int32, "U8": np.uint8, "BF16": "bf16"}


def read_safetensors(path: str) -> Dict[str, np.ndarray]:
    """Minimal safetensors reader (8-byte little-endian header length, JSON header, raw tensor bytes); BF16 is widened to f32."""
    with open(path, "rb") as f:
        n = struct.unpack("<Q", f.read(8))[0]
        if n > (1 << 28):
            raise ValueError("safetensors header is implausibly large")
        hdr = json.loads(f.read(n).decode("utf-8"))
        data = f.read()
    out = {}
    for name, info in hdr.items():
        if name == "__metadata__":
            continue
        b, e = info["data_offsets"]
        dt = _ST_DTYPES.get(info["dtype"])
        if dt is None:
            raise ValueError(f"tensor '{name}': unsupported safetensors dtype {info['dtype']}")
        if dt == "bf16":
            arr = gf.bf16_bits_to_f32(np.frombuffer(data, np.uint16, (e - b) // 2, b))
        else:
            arr = np.frombuffer(data, dt, (e - b) // np.dtype(dt).itemsize, b)
        out[name] = arr.reshape(info["shape"])
    return out


def write_safetensors(path: str, tensors: Dict[str, np.ndarray]) -> None:
    """Writer for tests (f32 / f16 tensors, insertion order)."""
    hdr, off, blobs = {}, 0, []
    for name, a in tensors.items():
        a = np.ascontiguousarray(a)
        dt = {np.dtype(np.float32): "F32", np.dtype(np.float16): "F16"}[a.dtype]
        hdr[name] = {"dtype": dt, "shape": list(a.shape), "data_offsets": [off, off + a.nbytes]}
        off += a.nbytes
        blobs.append(a.tobytes())
    js = json.dumps(hdr, separators=(",", ":")).encode()
    js += b" " * ((8 - len(js) % 8) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(js)))
        f.write(js)
        for b in blobs:
            f.write(b)


def load_state_dict(path: str) -> Dict[str, np.ndarray]:
    if path.endswith(".safetensors"):
        return read_safetensors(path)
    import torch  # checkpoints written by torch.save
    sd = torch.load(path, map_location="cpu", weights_only=True)
    for key in ("state_dict", "model"):
        if isinstance(sd, dict) and key in sd and isinstance(sd[key], dict):
            sd = sd[key]
    return {k: v.detach().to(torch.float32).numpy() for k, v in sd.items() if hasattr(v, "detach")}


def reg_token_count(sd: Dict[str, np.ndarray]) -> int:
    """R, the register tokens of a state dict ('reg_token' [1, R, D]; 0 without one)."""
    return int(sd["reg_token"].shape[1]) if "reg_token" in sd else 0


def infer_hparams(sd: Dict[str, np.ndarray], heads: Optional[int] = None):
    """(hidden, layers, heads, classes, patch, img, in_chans) from timm VisionTransformer tensor shapes."""
    pw = sd["patch_embed.proj.weight"]                       # (D, C, P, P)
    hidden, in_chans, patch = int(pw.shape[0]), int(pw.shape[1]), int(pw.shape[2])
    n_tok = int(sd["pos_embed"].shape[1])                    # (1, N, D), N = (img / patch)^2 + 1 + R, or (img / patch)^2 without cls_token
    R = reg_token_count(sd)
    prefix = 1 + R if "cls_token" in sd else 0
    grid = int(round(max(n_tok - prefix, 0) ** 0.5))
    if grid * grid + prefix != n_tok:
        raise ValueError(f"pos_embed has {n_tok} tokens: not a square patch grid" + (" plus one class token" if prefix else "") +
                         (f" and {R} registers" if R else ""))
    layers = 1 + max(int(m.group(1)) for k in sd for m in [re.match(r"blocks\.(\d+)\.", k)] if m)
    classes = int(sd["head.weight"].shape[0])
    heads = heads or hidden // 64
    if hidden % heads:
        raise ValueError(f"hidden size {hidden} is not divisible by {heads} heads")
    return hidden, layers, heads, classes, patch, grid * patch, in_chans


def resample_pos_embed(pos: np.ndarray, prefix: int, grid: int, antialias: bool = False) -> np.ndarray:
    """pos_embed [1, prefix + G^2, D] -> [1, prefix + grid^2, D]: the patch rows resampled on their square grid exactly as Hugging
    Face's interpolate_pos_encoding does it at run time (torch bicubic, align_corners False, in float32; Dinov2WithRegisters also
    antialiases), the `prefix` rows (class token, registers) kept."""
    import torch
    pos = np.asarray(pos, np.float32)
    D = pos.shape[-1]
    patches = pos.reshape(-1, D)[prefix:]
    G = int(round(len(patches) ** 0.5))
    if G * G != len(patches):
        raise ValueError(f"pos_embed has {len(patches)} patch rows: not a square grid")
    if G == grid:
        return pos
    t = torch.from_numpy(np.ascontiguousarray(patches.reshape(1, G, G, D).transpose(0, 3, 1, 2)))
    r = torch.nn.functional.interpolate(t, size=(grid, grid), mode="bicubic", align_corners=False, antialias=antialias)
    out = r.permute(0, 2, 3, 1).reshape(grid * grid, D).numpy()
    return np.concatenate([pos.reshape(-1, D)[:prefix], out]).reshape(1, -1, D).astype(np.float32)


def state_dict_to_model_file(sd: Dict[str, np.ndarray], out_path: str, ftype: int = 1, heads: Optional[int] = None,
                             id2label: Optional[Dict[int, str]] = None, container: str = "legacy", keep_norm_pre: bool = False,
                             activation: str = "gelu_tanh", eps: float = 1e-6, pool: str = "token", img_size: Optional[int] = None,
                             antialias: bool = False, image_proc: Optional[dict] = None) -> None:
    """keep_norm_pre, activation, eps: the architecture of a CLIP-pretrained timm ViT (norm_pre, QuickGELU or erf GELU, eps 1e-5);
    GGUF only.  Without them the file is the reference converter's, which drops norm_pre.  LayerScale ('blocks.{i}.ls1.gamma' /
    'ls2.gamma') and register tokens ('reg_token', with their R rows after the class row of pos_embed) are taken when the state dict has
    them; pool 'cls_patch_mean' makes the head read [class token || patch mean] (DINOv2's classifier); pools 'map' and 'mean' (SigLIP) are
    for a state dict without 'cls_token', 'map' with the 13 'attn_pool.*' tensors.  img_size: resample the patch position grid to
    img_size / patch (resample_pos_embed).  image_proc: a Hugging Face preprocessor_config.json dict, written as the vit.image_proc.* keys
    (GGUF only) after gf.image_proc_from_config has checked it against the model's input size."""
    assert ftype in (0, 1)
    layer_scale = int(any(k.endswith(".ls1.gamma") for k in sd))
    R = reg_token_count(sd)
    if pool not in gf.POOLS:
        raise ValueError(f"pool {pool!r} unknown ({', '.join(gf.POOLS)})")
    if container != "gguf" and (layer_scale or R or pool != "token"):
        raise ValueError("LayerScale, register tokens or another pool need --container gguf: a legacy ggml file carries the reference's "
                         "architecture only")
    if img_size is not None:
        # pools 'map' and 'mean' (SigLIP) take the floor grid of a size the patch does not divide, as HF's valid conv does
        P = int(sd["patch_embed.proj.weight"].shape[2])
        if img_size % P and pool not in ("map", "mean"):
            raise ValueError(f"img_size {img_size} is not a multiple of the patch size {P}")
        prefix = 1 + R if "cls_token" in sd else 0
        sd = dict(sd, pos_embed=resample_pos_embed(sd["pos_embed"], prefix, img_size // P, antialias))
    if activation not in gf.ARCH_ACTIVATIONS:
        raise ValueError(f"activation {activation!r} unknown ({', '.join(gf.ARCH_ACTIVATIONS)})")
    if container != "gguf" and (keep_norm_pre or activation != "gelu_tanh" or eps != 1e-6):
        raise ValueError("a pre-norm, another activation or another eps needs --container gguf: a legacy ggml file carries the "
                         "reference's architecture only")
    if container != "gguf" and image_proc is not None:
        raise ValueError("an image processor needs --container gguf: a legacy ggml file carries vit.cpp's preprocessing only")
    if keep_norm_pre and not ("norm_pre.weight" in sd and "norm_pre.bias" in sd):
        raise ValueError("keep_norm_pre: the state_dict has no norm_pre.weight / norm_pre.bias")
    hidden, layers, heads, classes, patch, img, in_chans = infer_hparams(sd, heads)
    img = img if img_size is None else img_size
    id2label = id2label or {i: f"LABEL_{i}" for i in range(classes)}   # convert-pth-to-ggml.py:95-96 fallback names
    vf = gf.VitFile(hidden, layers, heads, classes, patch, img, ftype, dict(id2label), eps=eps, pre_norm=int(keep_norm_pre),
                    activation=activation, layer_scale=layer_scale, reg_tokens=R, pool=pool,
                    image_proc=None if image_proc is None else gf.image_proc_from_config(image_proc, img))
    for k, v in sd.items():
        if k.startswith("norm_pre") and not keep_norm_pre:               # convert-pth-to-ggml.py:127-130
            continue
        a = np.asarray(v)
        if k == "patch_embed.proj.bias":
            a = a.reshape(1, a.shape[0], 1, 1)                           # convert-pth-to-ggml.py:150-151
        # convert-pth-to-ggml.py:143-147; the loader additionally hard-codes the patch kernel as F16 (vit.cpp:515), so an f32
        # file must still carry it as f16 (SURVEY.md 8c: the reference's own --ftype 0 output does not load)
        f16 = (ftype == 1 and np.asarray(v).ndim != 1 and k not in _F32_TOKENS) or k == "patch_embed.proj.weight"
        vf.tensors[k] = a.astype(np.float16 if f16 else np.float32)
        vf.tensor_ftype[k] = 1 if f16 else 0
    # vit.cpp:697, plus norm_pre.weight / .bias, the two LayerScale gammas of every block and reg_token; SigLIP's pools have no cls_token,
    # and the attention-pooling head 13 tensors
    expect = 4 + 12 * layers + 4 + 2 * vf.pre_norm + 2 * layers * layer_scale + (R > 0) - (pool in gf.PATCH_ONLY_POOLS) + 13 * (pool == "map")
    if len(vf.tensors) != expect:
        raise ValueError(f"state_dict has {len(vf.tensors)} tensors after filtering, a {layers}-layer ViT needs {expect}")
    if container == "gguf":
        gf.write_gguf(out_path, vf, "keep")
    else:
        write_legacy(out_path, vf)


# token rows and the pooling head's probe: kept f32 like every 1-D tensor
_F32_TOKENS = ("pos_embed", "cls_token", "reg_token", "attn_pool.latent")

# Hugging Face CLIP activations -> the file's (vitb200_arch.activation); HF's "gelu" is the erf form
_HF_ACTIVATIONS = {"quick_gelu": "quick_gelu", "gelu": "gelu_erf"}


def is_hf_clip(sd: Dict[str, np.ndarray]) -> bool:
    """A CLIPVisionModel, CLIPVisionModelWithProjection or CLIPModel state dict (the vision tower under `vision_model.`)."""
    return any(k.startswith("vision_model.") for k in sd)


def clip_to_timm(sd: Dict[str, np.ndarray], config: dict):
    """Hugging Face CLIP vision tower -> (timm VisionTransformer state dict in timm's key order, heads, activation, eps).
    config: the model's config.json (a CLIPConfig's `vision_config` is used when present).  The projection becomes the classifier
    head (bias 0), so the logits are HF's image_embeds; without one the head is the identity and the logits are the pooler_output.
    text_model.*, text_projection, logit_scale and position_ids are ignored."""
    vc = config.get("vision_config", config)
    act = vc.get("hidden_act", "quick_gelu")
    if act not in _HF_ACTIVATIONS:
        raise ValueError(f"hidden_act {act!r} is not supported (quick_gelu or gelu)")
    v = {k[len("vision_model."):]: np.asarray(a, np.float32) for k, a in sd.items() if k.startswith("vision_model.")}
    pw = v["embeddings.patch_embedding.weight"]                          # (D, C, P, P), no bias
    D = int(pw.shape[0])
    heads = int(vc.get("num_attention_heads", D // 64))
    if D % heads or D // heads not in (64, 80):  # 80: the ViT-H/14 towers (LAION-2B, DFN5B, MetaCLIP)
        raise ValueError(f"head dim {D / heads:g} is not supported (64 or 80)")
    layers = 1 + max(int(m.group(1)) for k in v for m in [re.match(r"encoder\.layers\.(\d+)\.", k)] if m)
    out = {
        "cls_token": v["embeddings.class_embedding"].reshape(1, 1, D),
        "pos_embed": v["embeddings.position_embedding.weight"].reshape(1, -1, D),
        "patch_embed.proj.weight": pw,
        "patch_embed.proj.bias": np.zeros(D, np.float32),
        "norm_pre.weight": v["pre_layrnorm.weight"],                     # HF's spelling
        "norm_pre.bias": v["pre_layrnorm.bias"],
    }
    hf_name = {"norm1": "layer_norm1", "attn.proj": "self_attn.out_proj", "norm2": "layer_norm2", "mlp.fc1": "mlp.fc1", "mlp.fc2": "mlp.fc2"}
    for i in range(layers):
        h, t = f"encoder.layers.{i}.", f"blocks.{i}."
        if v[h + "mlp.fc1.weight"].shape[0] != 4 * D:
            raise ValueError(f"intermediate size {v[h + 'mlp.fc1.weight'].shape[0]} is not supported (4 x hidden = {4 * D} only)")
        for dst in ("norm1", "attn.qkv", "attn.proj", "norm2", "mlp.fc1", "mlp.fc2"):  # timm's state_dict order
            for p in ("weight", "bias"):
                if dst == "attn.qkv":  # rows [q; k; v]
                    out[f"{t}{dst}.{p}"] = np.concatenate([v[f"{h}self_attn.{x}_proj.{p}"] for x in "qkv"], axis=0)
                else:
                    out[f"{t}{dst}.{p}"] = v[f"{h}{hf_name[dst]}.{p}"]
    out["norm.weight"], out["norm.bias"] = v["post_layernorm.weight"], v["post_layernorm.bias"]
    proj = sd.get("visual_projection.weight")
    out["head.weight"] = np.asarray(proj, np.float32) if proj is not None else np.eye(D, dtype=np.float32)
    out["head.bias"] = np.zeros(out["head.weight"].shape[0], np.float32)
    return out, heads, _HF_ACTIVATIONS[act], float(vc.get("layer_norm_eps", 1e-5))


def clip_to_model_file(sd: Dict[str, np.ndarray], config: dict, out_path: str, ftype: int = 1, id2label: Optional[Dict[int, str]] = None,
                       container: str = "gguf", image_proc: Optional[dict] = None) -> None:
    """A Hugging Face CLIP vision tower -> GGUF model file (pre-norm, the config's activation and eps)."""
    if container != "gguf":
        raise ValueError("a CLIP tower needs --container gguf: a legacy ggml file carries the reference's architecture only")
    tsd, heads, activation, eps = clip_to_timm(sd, config)
    state_dict_to_model_file(tsd, out_path, ftype, heads, id2label, "gguf", keep_norm_pre=True, activation=activation, eps=eps,
                             image_proc=image_proc)


_DINOV2_PREFIXES = ("dinov2.", "dinov2_with_registers.")


def is_hf_dinov2(sd: Dict[str, np.ndarray]) -> bool:
    """A Dinov2Model, Dinov2WithRegistersModel or their ForImageClassification state dict (keys unprefixed or under `dinov2.` /
    `dinov2_with_registers.`)."""
    return any(k.endswith("embeddings.patch_embeddings.projection.weight") for k in sd) and any(".layer_scale1.lambda1" in k for k in sd)


def dinov2_to_timm(sd: Dict[str, np.ndarray], config: dict):
    """Hugging Face DINOv2 -> (timm-named state dict, heads, activation, eps, pool, antialias).  query / key / value become attn.qkv,
    attention.output.dense attn.proj, layer_scale{1,2}.lambda1 ls{1,2}.gamma, embeddings.register_tokens reg_token (with R zero rows
    inserted into pos_embed after the class row: registers get no position embedding), layernorm norm; mask_token is dropped.  A
    classifier becomes the head with pool 'cls_patch_mean' (its logits are HF's); without one the head is the identity with pool 'token',
    so the logits are HF's pooler_output.  antialias: how HF resamples this class's position grid (Dinov2WithRegisters antialiases).
    use_swiglu_ffn (ViT-g): mlp.weights_in [2 F][D] becomes mlp.fc1 and mlp.weights_out [D][F] mlp.fc2, as they are, with activation
    'swiglu'; hidden_act and mlp_ratio are ignored, as HF ignores them, and F comes from the tensors."""
    swiglu = bool(config.get("use_swiglu_ffn", False))
    act = config.get("hidden_act", "gelu")
    if act != "gelu" and not swiglu:
        raise ValueError(f"hidden_act {act!r} is not supported (gelu only)")
    if not config.get("qkv_bias", True):
        raise ValueError("qkv_bias false is not supported (the engine's qkv has a bias)")
    if config.get("mlp_ratio", 4) != 4 and not swiglu:
        raise ValueError(f"mlp_ratio {config.get('mlp_ratio')} is not supported (4 only)")
    pre = next((p for p in _DINOV2_PREFIXES if any(k.startswith(p) for k in sd)), "")
    v = {k[len(pre):]: np.asarray(a, np.float32) for k, a in sd.items() if k.startswith(pre)}
    pw = v["embeddings.patch_embeddings.projection.weight"]            # (D, C, P, P)
    D = int(pw.shape[0])
    heads = int(config.get("num_attention_heads", D // 64))
    if D % heads or D // heads != 64:
        raise ValueError(f"head dim {D / heads:g} is not supported (64 only)")
    layers = 1 + max(int(m.group(1)) for k in v for m in [re.match(r"encoder\.layer\.(\d+)\.", k)] if m)
    reg = v.get("embeddings.register_tokens")
    R = 0 if reg is None else int(reg.shape[1])
    pos = v["embeddings.position_embeddings"].reshape(1, -1, D)
    out = {"cls_token": v["embeddings.cls_token"].reshape(1, 1, D),
           "pos_embed": np.concatenate([pos[:, :1], np.zeros((1, R, D), np.float32), pos[:, 1:]], axis=1),
           "patch_embed.proj.weight": pw, "patch_embed.proj.bias": v["embeddings.patch_embeddings.projection.bias"]}
    if R:
        out["reg_token"] = reg.reshape(1, R, D)
    for i in range(layers):
        h, t = f"encoder.layer.{i}.", f"blocks.{i}."
        if swiglu:
            if h + "mlp.weights_in.weight" not in v:
                raise ValueError(f"use_swiglu_ffn: the config asks for SwiGLU MLPs but block {i} has no mlp.weights_in")
        elif v[h + "mlp.fc1.weight"].shape[0] != 4 * D:
            raise ValueError(f"intermediate size {v[h + 'mlp.fc1.weight'].shape[0]} is not supported (4 x hidden = {4 * D} only)")
        for p in ("weight", "bias"):
            out[f"{t}norm1.{p}"] = v[f"{h}norm1.{p}"]
        for p in ("weight", "bias"):                                     # rows [q; k; v]
            out[f"{t}attn.qkv.{p}"] = np.concatenate([v[f"{h}attention.attention.{x}.{p}"] for x in ("query", "key", "value")], axis=0)
        for p in ("weight", "bias"):
            out[f"{t}attn.proj.{p}"] = v[f"{h}attention.output.dense.{p}"]
        out[f"{t}ls1.gamma"] = v[h + "layer_scale1.lambda1"]
        mlp = (("mlp.fc1", "mlp.weights_in"), ("mlp.fc2", "mlp.weights_out")) if swiglu else (("mlp.fc1", "mlp.fc1"), ("mlp.fc2", "mlp.fc2"))
        for dst, src in (("norm2", "norm2"),) + mlp:
            for p in ("weight", "bias"):
                out[f"{t}{dst}.{p}"] = v[f"{h}{src}.{p}"]
        out[f"{t}ls2.gamma"] = v[h + "layer_scale2.lambda1"]
    out["norm.weight"], out["norm.bias"] = v["layernorm.weight"], v["layernorm.bias"]
    cls_w = sd.get("classifier.weight")
    if cls_w is not None:
        out["head.weight"], out["head.bias"] = np.asarray(cls_w, np.float32), np.asarray(sd["classifier.bias"], np.float32)
    else:
        out["head.weight"], out["head.bias"] = np.eye(D, dtype=np.float32), np.zeros(D, np.float32)
    pool = "cls_patch_mean" if cls_w is not None else "token"
    return out, heads, "swiglu" if swiglu else "gelu_erf", float(config.get("layer_norm_eps", 1e-6)), pool, R > 0


def dinov2_to_model_file(sd: Dict[str, np.ndarray], config: dict, out_path: str, ftype: int = 1, id2label: Optional[Dict[int, str]] = None,
                         container: str = "gguf", img_size: Optional[int] = None, image_proc: Optional[dict] = None) -> None:
    """A Hugging Face DINOv2 -> GGUF model file (LayerScale, registers, erf GELU or SwiGLU, the config's eps; the classifier's pool)."""
    if container != "gguf":
        raise ValueError("a DINOv2 model needs --container gguf: a legacy ggml file carries the reference's architecture only")
    tsd, heads, activation, eps, pool, antialias = dinov2_to_timm(sd, config)
    if id2label is None and "id2label" in config and "classifier.weight" in sd:
        id2label = {int(k): str(x) for k, x in config["id2label"].items()}
    state_dict_to_model_file(tsd, out_path, ftype, heads, id2label, "gguf", activation=activation, eps=eps, pool=pool, img_size=img_size,
                             antialias=antialias, image_proc=image_proc)


def is_hf_siglip(sd: Dict[str, np.ndarray]) -> bool:
    """A SiglipVisionModel, SiglipModel or SiglipForImageClassification state dict: a CLIP-like vision tower (`vision_model.`) with a
    post_layernorm and position embeddings but no class embedding."""
    return ("vision_model.post_layernorm.weight" in sd and "vision_model.embeddings.position_embedding.weight" in sd and
            "vision_model.embeddings.class_embedding" not in sd)


def siglip_to_timm(sd: Dict[str, np.ndarray], config: dict):
    """Hugging Face SigLIP vision tower -> (timm-named state dict, heads, activation, eps, pool).  config: the model's config.json (a
    SiglipConfig's `vision_config` is used when present).  The token rows are the patches only (no cls_token).  Without a classifier the
    attention-pooling head becomes timm's AttentionPoolLatent tensors (head.probe -> attn_pool.latent, in_proj rows q -> attn_pool.q, k and
    v -> attn_pool.kv, out_proj -> attn_pool.proj, layernorm -> attn_pool.norm, mlp -> attn_pool.mlp) with pool 'map' and an identity
    head, so the logits are HF's pooler_output; SiglipForImageClassification's classifier becomes the head with pool 'mean' (its unused
    head.* is dropped).  text_model.*, logit_scale and logit_bias are ignored."""
    vc = config.get("vision_config", config)
    act = vc.get("hidden_act", "gelu_pytorch_tanh")
    if act != "gelu_pytorch_tanh":
        raise ValueError(f"hidden_act {act!r} is not supported (gelu_pytorch_tanh only)")
    v = {k[len("vision_model."):]: np.asarray(a, np.float32) for k, a in sd.items() if k.startswith("vision_model.")}
    pw = v["embeddings.patch_embedding.weight"]                          # (D, C, P, P)
    D = int(pw.shape[0])
    heads = int(vc.get("num_attention_heads", D // 64))
    if D % heads or D // heads not in (64, 72):
        raise ValueError(f"head dim {D / heads:g} is not supported (64, or 72 as So400m)")
    # the MLP width from the weights (So400m: 4304, not 4 D); a config that states another is refused
    F = int(v["encoder.layers.0.mlp.fc1.weight"].shape[0])
    inter = int(vc.get("intermediate_size", F))
    if inter != F:
        raise ValueError(f"intermediate_size {inter} is not supported: the weights' mlp.fc1 has {F} rows")
    # the input size: a patch that does not divide it drops the last pixel rows and columns (So400m at 384 px, 14-px patches: 27 x 27)
    P = int(pw.shape[2])
    n_pos = int(v["embeddings.position_embedding.weight"].shape[0])
    if "image_size" in vc and n_pos != (int(vc["image_size"]) // P) ** 2:
        raise ValueError(f"image_size {vc['image_size']}: {n_pos} position rows, not ({vc['image_size']} // {P})^2")
    classifier = "classifier.weight" in sd
    if not classifier and not vc.get("vision_use_head", True):
        raise ValueError("vision_use_head = false is not supported without a classifier: the tower's pooled output is its attention-pooling "
                         "head")
    layers = 1 + max(int(m.group(1)) for k in v for m in [re.match(r"encoder\.layers\.(\d+)\.", k)] if m)
    out = {"pos_embed": v["embeddings.position_embedding.weight"].reshape(1, -1, D), "patch_embed.proj.weight": pw,
           "patch_embed.proj.bias": v["embeddings.patch_embedding.bias"]}
    hf_name = {"norm1": "layer_norm1", "attn.proj": "self_attn.out_proj", "norm2": "layer_norm2", "mlp.fc1": "mlp.fc1", "mlp.fc2": "mlp.fc2"}
    for i in range(layers):
        h, t = f"encoder.layers.{i}.", f"blocks.{i}."
        if v[h + "mlp.fc1.weight"].shape[0] != F:
            raise ValueError(f"intermediate size {v[h + 'mlp.fc1.weight'].shape[0]} in block {i} is not supported (block 0's is {F})")
        for dst in ("norm1", "attn.qkv", "attn.proj", "norm2", "mlp.fc1", "mlp.fc2"):  # timm's state_dict order
            for p in ("weight", "bias"):
                if dst == "attn.qkv":  # rows [q; k; v]
                    out[f"{t}{dst}.{p}"] = np.concatenate([v[f"{h}self_attn.{x}_proj.{p}"] for x in "qkv"], axis=0)
                else:
                    out[f"{t}{dst}.{p}"] = v[f"{h}{hf_name[dst]}.{p}"]
    out["norm.weight"], out["norm.bias"] = v["post_layernorm.weight"], v["post_layernorm.bias"]
    if classifier:
        out["head.weight"], out["head.bias"] = np.asarray(sd["classifier.weight"], np.float32), np.asarray(sd["classifier.bias"], np.float32)
        return out, heads, act, float(vc.get("layer_norm_eps", 1e-6)), "mean"
    w, b = v["head.attention.in_proj_weight"], v["head.attention.in_proj_bias"]     # rows [q; k; v]
    out["attn_pool.latent"] = v["head.probe"].reshape(1, 1, D)
    out["attn_pool.q.weight"], out["attn_pool.q.bias"] = w[:D], b[:D]
    out["attn_pool.kv.weight"], out["attn_pool.kv.bias"] = w[D:], b[D:]
    for dst, src in (("proj", "attention.out_proj"), ("norm", "layernorm"), ("mlp.fc1", "mlp.fc1"), ("mlp.fc2", "mlp.fc2")):
        for p in ("weight", "bias"):
            out[f"attn_pool.{dst}.{p}"] = v[f"head.{src}.{p}"]
    out["head.weight"], out["head.bias"] = np.eye(D, dtype=np.float32), np.zeros(D, np.float32)
    return out, heads, act, float(vc.get("layer_norm_eps", 1e-6)), "map"


def siglip_to_model_file(sd: Dict[str, np.ndarray], config: dict, out_path: str, ftype: int = 1, id2label: Optional[Dict[int, str]] = None,
                         container: str = "gguf", image_proc: Optional[dict] = None) -> None:
    """A Hugging Face SigLIP vision tower -> GGUF model file (no class token, gelu_pytorch_tanh, the config's eps; pool 'map' or, with a
    classifier, 'mean').  img_size is the config's image_size (So400m-384: 384 with a 27 x 27 grid of 14-px patches), or the grid's
    pixels without one."""
    if container != "gguf":
        raise ValueError("a SigLIP tower needs --container gguf: a legacy ggml file carries the reference's architecture only")
    tsd, heads, activation, eps, pool = siglip_to_timm(sd, config)
    if id2label is None and "id2label" in config and "classifier.weight" in sd:
        id2label = {int(k): str(x) for k, x in config["id2label"].items()}
    img = config.get("vision_config", config).get("image_size")
    state_dict_to_model_file(tsd, out_path, ftype, heads, id2label, "gguf", activation=activation, eps=eps, pool=pool,
                             img_size=None if img is None else int(img), image_proc=image_proc)


# Hugging Face text activations -> the file's; HF's "gelu" is the erf form
_HF_TEXT_ACTIVATIONS = {"quick_gelu": "quick_gelu", "gelu": "gelu_erf", "gelu_pytorch_tanh": "gelu_pytorch_tanh"}
MAX_TEXT_CONTEXT = 224  # the split-precision attention's keys


def text_to_timm(sd: Dict[str, np.ndarray], config: dict):
    """The text tower (`text_model.*`) of a Hugging Face CLIP or SigLIP state dict -> (state dict in the engine's names, heads, activation,
    eps, text arch dict for VitFile.text).  config: config.json (a CLIPConfig's or SiglipConfig's `text_config` is used when present).
    SigLIP is recognised by its text head (`text_model.head.*`, the pooled row's projection with a bias) and pools the last row,
    bidirectionally; CLIP runs causally and pools the EOS row ('eos_argmax' when eos_token_id == 2, as HF does, 'eos' otherwise), with
    `text_projection` as the head (bias 0) or, for CLIPTextModel, the identity.  logit_scale / logit_bias are copied when present."""
    tc = config.get("text_config", config)
    v = {k[len("text_model."):]: np.asarray(a, np.float32) for k, a in sd.items() if k.startswith("text_model.")}
    if "embeddings.token_embedding.weight" not in v:
        raise ValueError("no text tower: the state dict has no text_model.embeddings.token_embedding.weight")
    siglip = "head.weight" in v
    act = tc.get("hidden_act", "gelu_pytorch_tanh" if siglip else "quick_gelu")
    if act not in _HF_TEXT_ACTIVATIONS:
        raise ValueError(f"hidden_act {act!r} is not supported ({', '.join(_HF_TEXT_ACTIVATIONS)})")
    tok = v["embeddings.token_embedding.weight"]                         # (V, D)
    D = int(tok.shape[1])
    heads = int(tc.get("num_attention_heads", D // 64))
    if D % heads or D // heads not in ((64, 72) if siglip else (64,)):
        raise ValueError(f"head dim {D / heads:g} is not supported (64; 72 in SigLIP towers)")
    # CLIP's MLP is 4 D; SigLIP's width is read from the weights (So400m: 4304)
    F = int(v["encoder.layers.0.mlp.fc1.weight"].shape[0]) if siglip else 4 * D
    pos = v["embeddings.position_embedding.weight"]                      # (N, D)
    if pos.shape[0] > MAX_TEXT_CONTEXT:
        raise ValueError(f"context {pos.shape[0]} is not supported (at most {MAX_TEXT_CONTEXT} tokens)")
    layers = 1 + max(int(m.group(1)) for k in v for m in [re.match(r"encoder\.layers\.(\d+)\.", k)] if m)
    out = {"token_embd.weight": tok, "pos_embed": pos.reshape(1, -1, D)}
    hf_name = {"norm1": "layer_norm1", "attn.proj": "self_attn.out_proj", "norm2": "layer_norm2", "mlp.fc1": "mlp.fc1", "mlp.fc2": "mlp.fc2"}
    for i in range(layers):
        h, t = f"encoder.layers.{i}.", f"blocks.{i}."
        if v[h + "mlp.fc1.weight"].shape[0] != F:
            raise ValueError(f"intermediate size {v[h + 'mlp.fc1.weight'].shape[0]} is not supported (" +
                             (f"block 0's is {F})" if siglip else f"4 x hidden = {4 * D} only)"))
        for dst in ("norm1", "attn.qkv", "attn.proj", "norm2", "mlp.fc1", "mlp.fc2"):
            for p in ("weight", "bias"):
                if dst == "attn.qkv":  # rows [q; k; v]
                    out[f"{t}{dst}.{p}"] = np.concatenate([v[f"{h}self_attn.{x}_proj.{p}"] for x in "qkv"], axis=0)
                else:
                    out[f"{t}{dst}.{p}"] = v[f"{h}{hf_name[dst]}.{p}"]
    out["norm.weight"], out["norm.bias"] = v["final_layer_norm.weight"], v["final_layer_norm.bias"]
    if siglip:
        out["head.weight"], out["head.bias"] = v["head.weight"], v["head.bias"]
    else:
        proj = sd.get("text_projection.weight")
        out["head.weight"] = np.asarray(proj, np.float32) if proj is not None else np.eye(D, dtype=np.float32)
        out["head.bias"] = np.zeros(out["head.weight"].shape[0], np.float32)
    eos = int(tc.get("eos_token_id", 2))
    scalar = lambda k: float(np.asarray(sd[k], np.float32).reshape(-1)[0]) if k in sd else None
    text = {"context": int(pos.shape[0]), "causal": 0 if siglip else 1, "pool": "last" if siglip else ("eos_argmax" if eos == 2 else "eos"),
            "eos_token_id": eos, "logit_scale": scalar("logit_scale"), "logit_bias": scalar("logit_bias")}
    return out, heads, _HF_TEXT_ACTIVATIONS[act], float(tc.get("layer_norm_eps", 1e-6 if siglip else 1e-5)), text


def text_to_model_file(sd: Dict[str, np.ndarray], config: dict, out_path: str, ftype: int = 1) -> None:
    """The text tower of a Hugging Face CLIP or SigLIP checkpoint -> GGUF text file (vitb200_create_text)."""
    tsd, heads, activation, eps, text = text_to_timm(sd, config)
    D, layers = int(tsd["token_embd.weight"].shape[1]), sum(1 for k in tsd if k.endswith(".norm1.weight"))
    vf = gf.VitFile(D, layers, heads, int(tsd["head.weight"].shape[0]), 0, 0, ftype, eps=eps, activation=activation, text=text)
    for k, a in tsd.items():
        f16 = ftype == 1 and a.ndim == 2  # the matrices; pos_embed [1, N, D] and every 1-D tensor stay f32
        vf.tensors[k] = np.asarray(a, np.float16 if f16 else np.float32)
        vf.tensor_ftype[k] = 1 if f16 else 0
    gf.write_gguf(out_path, vf, "keep")


def write_legacy(path: str, vf) -> None:
    """A VitFile (f32 / f16 / raw q8_0 tensors) -> legacy-ggml container, tensor order as stored."""
    with open(path, "wb") as f:
        f.write(struct.pack("i", gf.GGML_FILE_MAGIC))
        for v in (vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.num_classes, vf.patch_size, vf.img_size, vf.ftype):
            f.write(struct.pack("i", v))
        f.write(struct.pack("i", len(vf.id2label)))
        for key, value in vf.id2label.items():
            s = value.encode("utf-8")
            f.write(struct.pack("ii", key, len(s)))
            f.write(s)
        for name, arr in vf.tensors.items():
            if name.endswith(".q8_0_raw"):
                continue
            ft = vf.tensor_ftype[name]
            shape = arr.shape
            if name == "patch_embed.proj.bias" and arr.ndim == 1:
                shape = (1, arr.shape[0], 1, 1)                          # convert-pth-to-ggml.py:150-151
            nm = name.encode("utf-8")
            f.write(struct.pack("iii", len(shape), len(nm), ft))
            for d in reversed(shape):
                f.write(struct.pack("i", d))
            f.write(nm)
            if ft == 8:
                f.write(vf.tensors[name + ".q8_0_raw"].tobytes())
            else:
                np.ascontiguousarray(arr, np.float16 if ft == 1 else np.float32).tofile(f)


def quantize_q8_0_reference(x: np.ndarray) -> np.ndarray:
    """quantize_row_q8_0_reference (ggml-quants.c): per 32 values d = amax / 127 (stored f16), q = roundf(x * (1/d)), half away from
    zero.  x: float32 [n], n % 32 == 0.  Returns the raw block bytes (34 per block: f16 d, int8 q[32])."""
    x = np.ascontiguousarray(x, np.float32).reshape(-1, 32)
    amax = np.abs(x).max(axis=1)
    d = (amax / np.float32(127.0)).astype(np.float32)
    with np.errstate(divide="ignore"):
        inv = np.where(d != 0, np.float32(1.0) / d, np.float32(0.0)).astype(np.float32)
    x0 = (x * inv[:, None]).astype(np.float32)
    q = (np.sign(x0) * np.floor(np.abs(x0) + np.float32(0.5))).astype(np.int8)   # roundf
    out = np.empty((x.shape[0], 34), np.uint8)
    out[:, :2] = d.astype(np.float16).view(np.uint8).reshape(-1, 2)
    out[:, 2:] = q.view(np.uint8)
    return out.reshape(-1)


def quantize_model_file(src: str, dst: str, fmt: str = "q8_0") -> None:
    """reference quantize.cpp:26-330 for itype 8: every 2-D tensor whose name ends in `weight` is quantised row-wise, everything
    else is copied; the header's ftype becomes the quantisation type."""
    if fmt != "q8_0":
        raise ValueError("only q8_0 is restated here; the other block formats come from the reference's quantize binary")
    vf = gf.read(src)
    out = gf.VitFile(vf.hidden_size, vf.num_hidden_layers, vf.num_attention_heads, vf.num_classes, vf.patch_size, vf.img_size, 8,
                     dict(sorted(vf.id2label.items())))                  # quantize.cpp re-writes the labels from a std::map: key order
    for name, arr in vf.tensors.items():
        ft = vf.tensor_ftype[name]
        if name.endswith("weight") and arr.ndim == 2:                    # quantize.cpp:196-214
            out.tensors[name + ".q8_0_raw"] = quantize_q8_0_reference(arr.astype(np.float32))
            out.tensors[name] = arr
            out.tensor_ftype[name] = 8
        else:
            out.tensors[name] = arr
            out.tensor_ftype[name] = ft
    write_legacy(dst, out)


def add_image_proc(src: str, dst: str, preprocessor_config: dict) -> None:
    """A converted model file (GGUF, or the reference's legacy ggml with f32 / f16 tensors) -> GGUF with the vit.image_proc.* keys of a
    Hugging Face preprocessor_config.json dict; tensors and the other keys unchanged."""
    with open(src, "rb") as f:
        gguf = f.read(4) == gf.GGUF_MAGIC
    vf = gf.read_gguf(src) if gguf else gf.read(src)
    vf.image_proc = gf.image_proc_from_config(preprocessor_config, vf.img_size)
    gf.write_gguf(dst, vf, "keep")


def main(argv):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("src")
    ap.add_argument("dst")
    ap.add_argument("fmt", nargs="?", default="q8_0")
    ap.add_argument("--quantize", action="store_true")
    ap.add_argument("--ftype", type=int, choices=[0, 1], default=1)
    ap.add_argument("--heads", type=int, default=None)
    ap.add_argument("--labels", default=None, help="JSON file {class id: label}")
    ap.add_argument("--container", choices=["legacy", "gguf"], default=None,
                    help="default: legacy for the reference's architecture, gguf for a CLIP tower or the options below")
    ap.add_argument("--hf-config", default=None, help="config.json of a Hugging Face CLIP, DINOv2 or SigLIP checkpoint (required for one)")
    ap.add_argument("--keep-norm-pre", action="store_true", help="timm: keep norm_pre as the model's pre-norm (GGUF only)")
    ap.add_argument("--activation", choices=list(gf.ACTIVATIONS), default="gelu_tanh", help="timm: the MLP activation (GGUF only)")
    ap.add_argument("--eps", type=float, default=1e-6, help="timm: the LayerNorm epsilon (GGUF only)")
    ap.add_argument("--img-size", type=int, default=None,
                    help="resample the patch position embeddings to this input size (default: the checkpoint's grid)")
    ap.add_argument("--text", action="store_true", help="convert the text tower of a Hugging Face CLIP or SigLIP checkpoint (GGUF)")
    ap.add_argument("--hf-preprocessor", default=None,
                    help="preprocessor_config.json of a Hugging Face image processor: the u8 entry points prepare images as it does (GGUF)")
    a = ap.parse_args(argv)
    if a.quantize:
        quantize_model_file(a.src, a.dst, a.fmt)
        return
    labels = {int(k): v for k, v in json.load(open(a.labels)).items()} if a.labels else None
    proc = json.load(open(a.hf_preprocessor)) if a.hf_preprocessor else None
    with open(a.src, "rb") as f:
        magic = f.read(4)
    if proc is not None and (magic == gf.GGUF_MAGIC or magic == struct.pack("i", gf.GGML_FILE_MAGIC)):
        add_image_proc(a.src, a.dst, proc)
        return
    sd = load_state_dict(a.src)
    if a.text:
        if not a.hf_config:
            raise SystemExit("--text needs --hf-config <config.json> (hidden_act, layer_norm_eps, heads, eos_token_id)")
        text_to_model_file(sd, json.load(open(a.hf_config)), a.dst, a.ftype)
        return
    if is_hf_dinov2(sd):
        if not a.hf_config:
            raise SystemExit("a Hugging Face DINOv2 state dict needs --hf-config <config.json> (hidden_act, layer_norm_eps, heads)")
        dinov2_to_model_file(sd, json.load(open(a.hf_config)), a.dst, a.ftype, labels, a.container or "gguf", a.img_size, proc)
        return
    if is_hf_siglip(sd):
        if not a.hf_config:
            raise SystemExit("a Hugging Face SigLIP state dict needs --hf-config <config.json> (hidden_act, layer_norm_eps, heads)")
        if a.img_size:
            raise SystemExit("--img-size: resampling a SigLIP tower's position embeddings is not supported")
        siglip_to_model_file(sd, json.load(open(a.hf_config)), a.dst, a.ftype, labels, a.container or "gguf", proc)
        return
    if is_hf_clip(sd):
        if not a.hf_config:
            raise SystemExit("a Hugging Face CLIP state dict needs --hf-config <config.json> (hidden_act, layer_norm_eps, heads)")
        clip_to_model_file(sd, json.load(open(a.hf_config)), a.dst, a.ftype, labels, a.container or "gguf", proc)
        return
    new_arch = a.keep_norm_pre or a.activation != "gelu_tanh" or a.eps != 1e-6 or proc is not None
    state_dict_to_model_file(sd, a.dst, a.ftype, a.heads, labels, a.container or ("gguf" if new_arch else "legacy"),
                             a.keep_norm_pre, a.activation, a.eps, img_size=a.img_size, image_proc=proc)


if __name__ == "__main__":
    main(sys.argv[1:])
