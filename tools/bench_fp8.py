"""Dev tool (one H100): the FP8 engine (vitb200_create_from_file_fp8: qkv and fc1 on the e4m3 tensor cores) against the f16 engine.
Workloads: synthetic ViT-B/16 f16 at batch 256 and ViT-L/16-384 f16 at batch 128, seeded images resident on the device
(vitb200_forward_device, as bench.py times it).  Both engines live in one process; their windows of K forwards alternate over R
rounds (host clock from a synchronised device to a device synchronise), so clock and neighbour drift hit both alike.  Then, per
engine, one profiled window (vitb200_profile_*: CUDA events around every GEMM, attention and LayerNorm launch) for the per-kernel
table, with qkv and fc1 TFLOP/s against the data-sheet dense peaks (989 f16, 1979 FP8).  Last, the logit distance of the two engines
on the timed batch, max |FP8 - f16| / max |f16| per image, and their top-1 agreement.  The card name and power limit are read in
the same run.
usage: python tools/bench_fp8.py [--steps K] [--warmup W] [--rounds R] [--only base|large384]"""
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
# the tree may be read-only: generated model files go to a per-user temporary cache
os.environ.setdefault("VITB200_CACHE", os.path.join(tempfile.gettempdir(), "vitb200-cache-%d" % os.getuid()))
from tests.util import gf, model_path, pkg  # noqa: E402

eng = pkg.engine
KINDS = ["patch", "qkv", "proj", "fc1", "fc2", "head", "attention", "layernorm"]
PEAK_F16, PEAK_FP8 = 989.0, 1979.0  # TFLOP/s, dense, H100 SXM data sheet (700 W)
WORKLOADS = {"base": ("base", 256), "large384": ("large384", 128)}

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--only", choices=sorted(WORKLOADS), default=None)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_fp8.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


def card_info(index):
    """Name and power limit of the GPU the numbers were measured on (read-only query)."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        info["power_limit_w"] = float(out[0])
        info["max_sm_clock_mhz"] = float(out[1])
    except Exception as ex:
        info["power_limit_error"] = repr(ex)
    return info


def forward(m, d_img, B, d_probs, d_logits):
    rc = eng.lib().vitb200_forward_device(m.handle, d_img.data_ptr(), B, d_probs.data_ptr(),
                                          d_logits.data_ptr() if d_logits is not None else None, None, None, 0, None)
    if rc:
        raise RuntimeError(eng.lib().vitb200_last_error().decode())


def window(m, d_img, B, d_probs, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        forward(m, d_img, B, d_probs, None)
    torch.cuda.synchronize()
    return B * steps / (time.perf_counter() - t0)


def profile(m, d_img, B, d_probs, steps):
    L = eng.lib()
    L.vitb200_profile_enable(m.handle, 1)
    for _ in range(steps):
        forward(m, d_img, B, d_probs, None)
    rows = {}
    for k, name in enumerate(KINDS):
        ms, n, fl = C.c_double(), C.c_int(), C.c_double()
        L.vitb200_profile_read(m.handle, k, C.byref(ms), C.byref(n), C.byref(fl))
        per_step = ms.value / steps
        rows[name] = {"ms_per_step": round(per_step, 3)}
        if fl.value > 0 and n.value:
            rows[name]["tflops"] = round(fl.value * n.value / (ms.value * 1e-3) / 1e12, 1)
    L.vitb200_profile_enable(m.handle, 0)
    return rows


def run(cfg, B):
    path = model_path(cfg, "f16")
    S = gf.CONFIGS[cfg][4]
    d_img = torch.from_numpy(gf.synthetic_images(B, S, seed=2024)).cuda()
    models = {"f16": eng.vit_model_load(path, 0, B), "fp8": eng.vit_model_load(path, 0, B, fp8=True)}
    assert models["fp8"].fp8 and not models["f16"].fp8
    nc = models["f16"].num_classes
    d_probs = torch.empty((B, nc), dtype=torch.float32, device="cuda")
    for m in models.values():
        window(m, d_img, B, d_probs, args.warmup)
    rates = {k: [] for k in models}
    for _ in range(args.rounds):
        for k, m in models.items():
            rates[k].append(round(window(m, d_img, B, d_probs, args.steps), 1))
    prof = {k: profile(m, d_img, B, d_probs, args.steps) for k, m in models.items()}
    for k, peak in (("f16", PEAK_F16), ("fp8", PEAK_FP8)):
        for g in ("qkv", "fc1"):
            if "tflops" in prof[k][g]:
                prof[k][g]["share_of_peak"] = round(prof[k][g]["tflops"] / peak, 3)
    logits = {}
    for k, m in models.items():
        d_l = torch.empty((B, nc), dtype=torch.float32, device="cuda")
        forward(m, d_img, B, d_probs, d_l)
        torch.cuda.synchronize()
        logits[k] = d_l.cpu().numpy()
        m.close()
    a, b = logits["fp8"].astype(np.float64), logits["f16"].astype(np.float64)
    dist = np.abs(a - b).max(axis=1) / np.abs(b).max(axis=1)
    med = {k: float(np.median(v)) for k, v in rates.items()}
    return {
        "workload": f"{cfg} f16 file, batch {B}",
        "images_per_s": rates, "median_images_per_s": med, "fp8_over_f16": round(med["fp8"] / med["f16"], 3),
        "per_kernel": prof,
        "logit_dist_fp8_vs_f16": {"median": float(np.median(dist)), "max": float(dist.max())},
        "top1_agreement": float((a.argmax(1) == b.argmax(1)).mean()),
    }


out = {"card": card_info(0), "steps": args.steps, "rounds": args.rounds, "results": []}
for name, (cfg, B) in WORKLOADS.items():
    if args.only and name != args.only:
        continue
    out["results"].append(run(cfg, B))
    print(json.dumps(out["results"][-1]), flush=True)
print(json.dumps({"card": out["card"]}), flush=True)
