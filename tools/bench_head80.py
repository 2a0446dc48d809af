"""Dev tool (one H100): ViT-H/14's 80-column attention heads against 64-column heads at the same width.
Two seeded synthetic models of the same shape -- D 1280, 32 layers, patch 14, 224 px (257 tokens), 1000 classes -- one with 16 heads of
80 columns (ViT-H/14) and one with 20 heads of 64, at batch 128, images resident on the device.  Both do the same attention FLOPs
(4 N^2 D per image per layer); the head-dim-80 model computes 4/5 as many soft-max exponentials.  Above 224 tokens the head-dim-80 model
runs attention_hd80_kernel on f16 operands and the head-dim-64 one the 16-warp attention_kernel.
    1. images/s of vitb200_forward_device over R rounds of K calls, alternating the two models in one process (host clock from a
       synchronised device to a device synchronise);
    2. a separate profiled pass per model (vitb200_profile_*): attention ms per step and TFLOP/s, and the step's other kernel kinds.
The card name, power limit and max SM clock are read in the same run.
usage: python tools/bench_head80.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
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
D, L, P, S, CLASSES = 1280, 32, 14, 224, 1000
HEADS = {"hd80": 16, "hd64": 20}

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=128)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_head80.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


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


def model_file(directory, heads):
    """A seeded synthetic ViT (ggml_file.synth_tensors, the same weights for both head counts), GGUF with f16 matrices."""
    vf = gf.VitFile(D, L, heads, CLASSES, P, S, 1)
    for name, arr in gf.synth_tensors(D, L, CLASSES, P, S, seed=7).items():
        f16 = arr.ndim >= 2 and name not in ("cls_token", "pos_embed")
        if name == "patch_embed.proj.bias":
            arr = arr.reshape(1, -1, 1, 1)  # the conv bias's declared shape, as convert.py writes it
        vf.tensors[name] = arr.astype(np.float16 if f16 else np.float32)
        vf.tensor_ftype[name] = 1 if f16 else 0
    path = os.path.join(directory, f"h{heads}.gguf")
    gf.write_gguf(path, vf)
    return path


def check(rc):
    if rc:
        raise RuntimeError(eng.lib().vitb200_last_error().decode())


def main():
    B = args.batch
    N = (S // P) ** 2 + 1
    tmp = tempfile.mkdtemp(prefix="bench_head80_")
    models = {k: eng.vit_model_load(model_file(tmp, h), 0, B) for k, h in HEADS.items()}
    d_img = torch.from_numpy(gf.synthetic_images(B, S, seed=2024)).cuda()
    d_logits = torch.empty((B, CLASSES), dtype=torch.float32, device="cuda")
    Lb = eng.lib()

    def call(m):
        check(Lb.vitb200_forward_device(m.handle, d_img.data_ptr(), B, None, d_logits.data_ptr(), None, None, 0, None))

    def window(m, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            call(m)
        torch.cuda.synchronize()
        return B * steps / (time.perf_counter() - t0)

    out = {"card": card_info(0), "shape": f"D {D}, {L} layers, {N} tokens, batch {B}", "steps": args.steps, "rounds": args.rounds}
    for m in models.values():
        window(m, args.warmup)
    rates = {k: [] for k in models}
    for _ in range(args.rounds):
        for k, m in models.items():
            rates[k].append(round(window(m, args.steps), 1))
    out["images_per_s"] = rates
    out["images_per_s_median"] = {k: float(np.median(v)) for k, v in rates.items()}
    prof = {}
    for k, m in models.items():
        Lb.vitb200_profile_enable(m.handle, 1)
        for _ in range(args.steps):
            call(m)
        torch.cuda.synchronize()
        prof[k] = {}
        for kind, name in enumerate(KINDS):
            ms, cnt, fl = C.c_double(), C.c_int(), C.c_double()
            check(Lb.vitb200_profile_read(m.handle, kind, C.byref(ms), C.byref(cnt), C.byref(fl)))
            if cnt.value:
                per_step = ms.value / args.steps
                prof[k][name] = {"ms_per_step": round(per_step, 3), "launches_per_step": cnt.value // args.steps}
                if fl.value:
                    prof[k][name]["tflops"] = round(fl.value * cnt.value / (ms.value * 1e-3) / 1e12, 1)
        Lb.vitb200_profile_enable(m.handle, 0)
        # the attention's FLOPs as the engine counts them: 4 N^2 D per image per layer, whatever the head dim
        assert prof[k]["attention"]["launches_per_step"] == L
    out["profile"] = prof
    out["attention_flops_per_step"] = 4.0 * B * L * N * N * D
    for m in models.values():
        m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
