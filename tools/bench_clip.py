"""Dev tool (one H100): the cost of the CLIP architecture (vitb200_arch: pre-norm + QuickGELU) on an L/14-336-shaped tower.
Two synthetic models of the same shape -- 24 layers, D 1024, 16 heads, patch 14, 336 px (577 tokens), 768 outputs -- one with the
reference's architecture (tanh GELU, no pre-norm) and one CLIP tower (pre-norm, QuickGELU, eps 1e-5), at batch 128, images resident on
the device.  Two workloads, each alternating the two models over R rounds of K calls (host clock from a synchronised device to a device
synchronise), in one process:
    llava   vitb200_features_device at layers = 23, norm = 0, f16 tokens (LLaVA's image features)
    embeds  vitb200_forward_device, logits = the image embeddings
Then one profiled window per model (vitb200_profile_*) for fc1's and the LayerNorms' ms per step.  The card name and power limit are read
in the same run.
usage: python tools/bench_clip.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
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
SHAPE = (1024, 24, 16, 14, 336)  # hidden, layers, heads, patch, img
PROJ = 768

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=128)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_clip.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


def card_info(index):
    """Name and power limit of the GPU the numbers were measured on (read-only query)."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit_w"] = float(out)
    except Exception as ex:
        info["power_limit_error"] = repr(ex)
    return info


def model_file(directory, clip):
    """A seeded synthetic tower (ggml_file.synth_tensors); the CLIP one adds norm_pre and its architecture keys.  GGUF, f16 matrices."""
    D, L, H, P, S = SHAPE
    vf = gf.VitFile(D, L, H, PROJ, P, S, 1)
    for name, arr in gf.synth_tensors(D, L, PROJ, P, S, seed=7).items():
        f16 = arr.ndim >= 2 and name not in ("cls_token", "pos_embed")
        if name == "patch_embed.proj.bias":
            arr = arr.reshape(1, -1, 1, 1)  # the conv bias's declared shape, as convert.py writes it
        vf.tensors[name] = arr.astype(np.float16 if f16 else np.float32)
        vf.tensor_ftype[name] = 1 if f16 else 0
    if clip:
        rng = np.random.default_rng(8)
        vf.tensors["norm_pre.weight"] = (1 + 0.02 * rng.standard_normal(D)).astype(np.float32)
        vf.tensors["norm_pre.bias"] = (0.02 * rng.standard_normal(D)).astype(np.float32)
        vf.tensor_ftype["norm_pre.weight"] = vf.tensor_ftype["norm_pre.bias"] = 0
        vf.pre_norm, vf.activation, vf.eps = 1, "quick_gelu", 1e-5
    path = os.path.join(directory, "clip.gguf" if clip else "ref.gguf")
    gf.write_gguf(path, vf)
    return path


def check(rc):
    if rc:
        raise RuntimeError(eng.lib().vitb200_last_error().decode())


def main():
    B = args.batch
    tmp = tempfile.mkdtemp(prefix="bench_clip_")
    models = {k: eng.vit_model_load(model_file(tmp, k == "clip"), 0, B) for k in ("reference", "clip")}
    assert models["clip"].arch == {"pre_norm": True, "activation": "quick_gelu"}
    D, L = SHAPE[0], SHAPE[1]
    N = (SHAPE[4] // SHAPE[3]) ** 2 + 1
    d_img = torch.from_numpy(gf.synthetic_images(B, SHAPE[4], seed=2024)).cuda()
    d_tok = torch.empty((B, N, D), dtype=torch.float16, device="cuda")
    d_logits = torch.empty((B, PROJ), dtype=torch.float32, device="cuda")
    req = eng.FeaturesReq(L - 1, 0, 1)
    Lb = eng.lib()
    calls = {
        "llava": lambda m: check(Lb.vitb200_features_device(m.handle, d_img.data_ptr(), B, C.byref(req), d_tok.data_ptr(), None, None)),
        "embeds": lambda m: check(Lb.vitb200_forward_device(m.handle, d_img.data_ptr(), B, None, d_logits.data_ptr(), None, None, 0, None)),
    }

    def window(m, call, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            call(m)
        torch.cuda.synchronize()
        return B * steps / (time.perf_counter() - t0)

    out = {"card": card_info(0), "shape": "L/14-336 (24 layers, 577 tokens)", "batch": B, "steps": args.steps, "rounds": args.rounds}
    for wl, call in calls.items():
        for m in models.values():
            window(m, call, args.warmup)
        rates = {k: [] for k in models}
        for _ in range(args.rounds):
            for k, m in models.items():
                rates[k].append(round(window(m, call, args.steps), 1))
        med = {k: float(np.median(v)) for k, v in rates.items()}
        prof = {}
        for k, m in models.items():
            Lb.vitb200_profile_enable(m.handle, 1)
            for _ in range(args.steps):
                call(m)
            prof[k] = {}
            for kind in ("fc1", "layernorm"):
                ms, n, fl = C.c_double(), C.c_int(), C.c_double()
                check(Lb.vitb200_profile_read(m.handle, KINDS.index(kind), C.byref(ms), C.byref(n), C.byref(fl)))
                prof[k][kind] = {"ms_per_step": round(ms.value / args.steps, 3), "launches_per_step": n.value // args.steps}
            Lb.vitb200_profile_enable(m.handle, 0)
        out[wl] = {"images_per_s": rates, "median_images_per_s": med, "clip_over_reference": round(med["clip"] / med["reference"], 4),
                   "profiled": prof}
        print(json.dumps({wl: out[wl]}), flush=True)
    for m in models.values():
        m.close()
    print(json.dumps(out), flush=True)


main()
