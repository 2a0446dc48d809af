"""Dev tool (one H100): the cost of SwiGLU MLPs (vitb200_arch.activation = 4, the gate fused into the fc1 epilogue) on DINOv2 ViT-g/14.
Two seeded synthetic models of the same D, L and heads -- 40 layers, D 1536, 24 heads, patch 14, 224 px, 1000 classes -- built from
tensors with vit_model_from_tensors (no 2 GB file): a ViT-g/14 DINOv2 classifier (SwiGLU F = 4096, LayerScale, 4 registers: 261 tokens,
the head reads [LN(cls) || mean LN(patches)]) and a reference-architecture model (tanh GELU, F = 6144: 257 tokens).  At batch 128, images
resident on the device, vitb200_forward_device (logits) alternates the two models over R rounds of K calls (host clock from a
synchronised device to a device synchronise), in one process; then one profiled window per model (vitb200_profile_*) gives fc1's and
fc2's ms per step and each fc1's achieved TFLOP/s from its algorithmic FLOPs (2 T 2F D for SwiGLU, 2 T F D for GELU).  The card name,
power limit and max SM clock are read in the same run.  About 10 GB of host memory at peak.
usage: python tools/bench_swiglu.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.util import gf, pkg  # noqa: E402

eng = pkg.engine
KINDS = ["patch", "qkv", "proj", "fc1", "fc2", "head", "attention", "layernorm"]
SHAPE = (1536, 40, 24, 14, 224)  # hidden, layers, heads, patch, img
CLASSES, REG, F = 1000, 4, 4096

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=128)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_swiglu.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


def card_info(index):
    """Name, power limit and max SM clock of the GPU the numbers were measured on (read-only query)."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        pl, clk = (x.strip() for x in out.split(","))
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(pl), float(clk)
    except Exception as ex:
        info["query_error"] = repr(ex)
    return info


def model(swiglu):
    """A seeded synthetic VitFile, f16 matrices generated tensor by tensor (float32 normals, then f16): the reference's tensors, or the
    ViT-g classifier's (fc1 [2 F][D], fc2 [D][F], gammas, registers, a 2 D head)."""
    D, L, H, P, S = SHAPE
    vf = gf.VitFile(D, L, H, CLASSES, P, S, 1)
    rng = np.random.default_rng(7)
    for name, shape, is_mat in gf.tensor_specs(D, L, CLASSES, P, S, 3):
        if swiglu and name.endswith("mlp.fc1.weight"):
            shape = (2 * F, D)
        elif swiglu and name.endswith("mlp.fc1.bias"):
            shape = (2 * F,)
        elif swiglu and name.endswith("mlp.fc2.weight"):
            shape = (D, F)
        elif swiglu and name == "pos_embed":
            shape = (1, shape[1] + REG, D)
        elif swiglu and name == "head.weight":
            shape = (CLASSES, 2 * D)
        scale = 1.0 / np.sqrt(shape[-1]) if is_mat and name != "patch_embed.proj.weight" else 0.02
        a = rng.standard_normal(shape, dtype=np.float32) * np.float32(scale)
        if name.endswith(("norm1.weight", "norm2.weight")) or name == "norm.weight":
            a += np.float32(1.0)
        f16 = a.ndim >= 2 and name not in ("cls_token", "pos_embed")
        vf.tensors[name] = a.astype(np.float16) if f16 else a
        vf.tensor_ftype[name] = 1 if f16 else 0
    if swiglu:
        for i in range(L):
            for g in ("ls1", "ls2"):
                vf.tensors[f"blocks.{i}.{g}.gamma"] = np.exp(rng.uniform(np.log(1e-5), 0.0, D)).astype(np.float32)
                vf.tensor_ftype[f"blocks.{i}.{g}.gamma"] = 0
        vf.tensors["reg_token"] = (0.5 * rng.standard_normal((1, REG, D))).astype(np.float32)
        vf.tensor_ftype["reg_token"] = 0
        vf.activation, vf.layer_scale, vf.reg_tokens, vf.pool = "swiglu", 1, REG, "cls_patch_mean"
    return vf


def check(rc):
    if rc:
        raise RuntimeError(eng.lib().vitb200_last_error().decode())


def main():
    B = args.batch
    models = {}
    for k in ("gelu", "swiglu"):
        vf = model(k == "swiglu")
        models[k] = eng.vit_model_from_tensors(vf, 0, B)
        del vf
    assert models["swiglu"].arch["activation"] == "swiglu" and models["swiglu"].mlp_dim == F and models["gelu"].mlp_dim == 4 * SHAPE[0]
    d_img = torch.from_numpy(gf.synthetic_images(B, SHAPE[4], seed=2024)).cuda()
    d_logits = torch.empty((B, CLASSES), dtype=torch.float32, device="cuda")
    Lb = eng.lib()
    call = lambda m: check(Lb.vitb200_forward_device(m.handle, d_img.data_ptr(), B, None, d_logits.data_ptr(), None, None, 0, None))

    def window(m, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            call(m)
        torch.cuda.synchronize()
        return B * steps / (time.perf_counter() - t0)

    out = {"card": card_info(0), "shape": "ViT-g/14 at 224 (40 layers, D 1536; 261 tokens with 4 registers, 257 without)", "batch": B,
           "steps": args.steps, "rounds": args.rounds}
    for m in models.values():
        window(m, args.warmup)
    rates = {k: [] for k in models}
    for _ in range(args.rounds):
        for k, m in models.items():
            rates[k].append(round(window(m, args.steps), 1))
    med = {k: float(np.median(v)) for k, v in rates.items()}
    prof = {}
    for k, m in models.items():
        Lb.vitb200_profile_enable(m.handle, 1)
        for _ in range(args.steps):
            call(m)
        prof[k] = {}
        for kind in KINDS:
            ms, n, fl = C.c_double(), C.c_int(), C.c_double()
            check(Lb.vitb200_profile_read(m.handle, KINDS.index(kind), C.byref(ms), C.byref(n), C.byref(fl)))
            r = {"ms_per_step": round(ms.value / args.steps, 3), "launches_per_step": n.value // args.steps}
            if kind in ("fc1", "fc2") and ms.value > 0:
                r["tflops"] = round(fl.value * n.value / (ms.value * 1e-3) / 1e12, 1)
            prof[k][kind] = r
        Lb.vitb200_profile_enable(m.handle, 0)
        prof[k]["launches"] = m.last_launch_count()
    out.update({"images_per_s": rates, "median_images_per_s": med, "swiglu_over_gelu": round(med["swiglu"] / med["gelu"], 4),
                "fc1_tflops_swiglu_over_gelu": round(prof["swiglu"]["fc1"]["tflops"] / prof["gelu"]["fc1"]["tflops"], 4),
                "profiled": prof})
    for m in models.values():
        m.close()
    print(json.dumps(out), flush=True)


main()
