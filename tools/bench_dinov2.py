"""Dev tool (one H100): the cost of DINOv2's architecture (vitb200_arch: LayerScale in the proj / fc2 epilogues, 4 register tokens, the
class-plus-patch-mean pool) on a B/14 classifier at 224 px.
Two synthetic seeded models of the same shape -- 12 layers, D 768, 12 heads, patch 14, 224 px, 1000 classes -- one with the
reference's architecture (257 tokens) and one DINOv2 classifier with registers (erf GELU, LayerScale, 4 registers: 261 tokens, the head
reads [LN(cls) || mean LN(patches)], K = 2 D), at batch 256, images resident on the device.  vitb200_forward_device (logits) alternates
the two models over R rounds of K calls (host clock from a synchronised device to a device synchronise), in one process; then one
profiled window per model (vitb200_profile_*) gives proj's, fc2's, the LayerNorms' (the pool included) and the head's ms per step.  The
card name, power limit and max SM clock are read in the same run.
usage: python tools/bench_dinov2.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.util import gf, pkg  # noqa: E402

eng = pkg.engine
KINDS = ["patch", "qkv", "proj", "fc1", "fc2", "head", "attention", "layernorm"]
SHAPE = (768, 12, 12, 14, 224)  # hidden, layers, heads, patch, img
CLASSES, REG = 1000, 4

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=256)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_dinov2.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


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


def model_file(directory, dino):
    """A seeded synthetic model (ggml_file.synth_tensors); the DINOv2 one adds gammas, registers and a 2 D head.  GGUF, f16 matrices."""
    D, L, H, P, S = SHAPE
    vf = gf.VitFile(D, L, H, CLASSES, P, S, 1)
    rng = np.random.default_rng(8)
    for name, arr in gf.synth_tensors(D, L, CLASSES, P, S, seed=7).items():
        if dino and name == "pos_embed":
            arr = np.concatenate([arr[:, :1], np.zeros((1, REG, D), arr.dtype), arr[:, 1:]], axis=1)
        if dino and name == "head.weight":
            arr = np.concatenate([arr, arr[:, ::-1]], axis=1) * np.float32(0.5 ** 0.5)
        f16 = arr.ndim >= 2 and name not in ("cls_token", "pos_embed")
        if name == "patch_embed.proj.bias":
            arr = arr.reshape(1, -1, 1, 1)
        vf.tensors[name] = arr.astype(np.float16 if f16 else np.float32)
        vf.tensor_ftype[name] = 1 if f16 else 0
    if dino:
        for i in range(L):
            for g in ("ls1", "ls2"):
                vf.tensors[f"blocks.{i}.{g}.gamma"] = np.exp(rng.uniform(np.log(1e-5), 0.0, D)).astype(np.float32)
                vf.tensor_ftype[f"blocks.{i}.{g}.gamma"] = 0
        vf.tensors["reg_token"] = (0.5 * rng.standard_normal((1, REG, D))).astype(np.float32)
        vf.tensor_ftype["reg_token"] = 0
        vf.activation, vf.layer_scale, vf.reg_tokens, vf.pool = "gelu_erf", 1, REG, "cls_patch_mean"
    path = os.path.join(directory, "dinov2.gguf" if dino else "ref.gguf")
    gf.write_gguf(path, vf)
    return path


def check(rc):
    if rc:
        raise RuntimeError(eng.lib().vitb200_last_error().decode())


def main():
    B = args.batch
    tmp = tempfile.mkdtemp(prefix="bench_dinov2_")
    models = {k: eng.vit_model_load(model_file(tmp, k == "dinov2"), 0, B) for k in ("reference", "dinov2")}
    assert (models["dinov2"].layer_scale, models["dinov2"].reg_tokens, models["dinov2"].pool) == (True, REG, "cls_patch_mean")
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

    out = {"card": card_info(0), "shape": "B/14 at 224 (12 layers; 257 tokens, 261 with 4 registers)", "batch": B, "steps": args.steps,
           "rounds": args.rounds}
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
            prof[k][kind] = {"ms_per_step": round(ms.value / args.steps, 3), "launches_per_step": n.value // args.steps}
        Lb.vitb200_profile_enable(m.handle, 0)
        prof[k]["launches"] = m.last_launch_count()
    out.update({"images_per_s": rates, "median_images_per_s": med, "dinov2_over_reference": round(med["dinov2"] / med["reference"], 4),
                "profiled": prof})
    for m in models.values():
        m.close()
    print(json.dumps(out), flush=True)


main()
