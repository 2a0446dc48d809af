"""Dev tool (one H100): the cost of SigLIP's architecture (vitb200_arch pool 2: patch-only token rows, the attention-pooling head;
activation 3: PyTorch's tanh GELU in fc1) against the reference architecture of the same shape.
Two pairs of synthetic seeded models, 1000 classes, GGUF with f16 matrices, images resident on the device:
    B/16 at 224, 12 layers, batch 256: the reference architecture (197 tokens) and a SigLIP MAP tower (196 tokens)
    L/16 at 384, 24 layers, batch 128: the reference architecture (large384, 577 tokens) and a SigLIP MAP tower (576 tokens)
vitb200_forward_device (logits) alternates the two models of a pair over R rounds of K calls (host clock from a synchronised device to a
device synchronise), in one process; then one profiled window per model (vitb200_profile_*) gives every kernel kind's ms per step, kind 8
(the pooling head) included, and fc1 under activation 3 against activation 0.  A torch.profiler window per SigLIP model times
attention_pool_kernel alone, against its HBM bound: 4 P D bytes per image (k and v, f16) at the data sheet's 3.35 TB/s.  The card name,
power limit and max SM clock are read in the same run.
usage: python tools/bench_siglip.py [--steps K] [--warmup W] [--rounds R]"""
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
KINDS = ["patch", "qkv", "proj", "fc1", "fc2", "head", "attention", "layernorm", "pool_head"]
PAIRS = {"B/16-224": ((768, 12, 12, 16, 224), 256), "L/16-384": ((1024, 24, 16, 16, 384), 128)}
CLASSES = 1000
HBM_BYTES_PER_S = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_siglip.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


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


def model_file(directory, shape, siglip):
    """A seeded synthetic model (ggml_file.synth_tensors); the SigLIP one drops the class token and its position row and adds the 13
    attention-pooling head tensors."""
    D, L, H, P, S = shape
    vf = gf.VitFile(D, L, H, CLASSES, P, S, 1)
    rng = np.random.default_rng(8)
    for name, arr in gf.synth_tensors(D, L, CLASSES, P, S, seed=7).items():
        if siglip and name == "cls_token":
            continue
        if siglip and name == "pos_embed":
            arr = arr[:, 1:]
        f16 = arr.ndim >= 2 and name not in ("cls_token", "pos_embed")
        if name == "patch_embed.proj.bias":
            arr = arr.reshape(1, -1, 1, 1)
        vf.tensors[name] = arr.astype(np.float16 if f16 else np.float32)
        vf.tensor_ftype[name] = 1 if f16 else 0
    if siglip:
        head = {"attn_pool.latent": (1, 1, D), "attn_pool.q.weight": (D, D), "attn_pool.q.bias": (D,), "attn_pool.kv.weight": (2 * D, D),
                "attn_pool.kv.bias": (2 * D,), "attn_pool.proj.weight": (D, D), "attn_pool.proj.bias": (D,), "attn_pool.norm.weight": (D,),
                "attn_pool.norm.bias": (D,), "attn_pool.mlp.fc1.weight": (4 * D, D), "attn_pool.mlp.fc1.bias": (4 * D,),
                "attn_pool.mlp.fc2.weight": (D, 4 * D), "attn_pool.mlp.fc2.bias": (D,)}
        for name, shp in head.items():
            mat = len(shp) == 2
            a = rng.standard_normal(shp) * (shp[-1] ** -0.5 if mat else 0.05)
            if name == "attn_pool.norm.weight":
                a = 1.0 + a
            vf.tensors[name] = a.astype(np.float16 if mat else np.float32)
            vf.tensor_ftype[name] = 1 if mat else 0
        vf.activation, vf.pool = "gelu_pytorch_tanh", "map"
    path = os.path.join(directory, f"{'siglip' if siglip else 'ref'}-{D}-{L}.gguf")
    gf.write_gguf(path, vf)
    return path


def check(rc):
    if rc:
        raise RuntimeError(eng.lib().vitb200_last_error().decode())


def run_pair(tmp, label, shape, B):
    D, L, H, P, S = shape
    models = {k: eng.vit_model_load(model_file(tmp, shape, k == "siglip"), 0, B) for k in ("reference", "siglip")}
    assert models["siglip"].pool == "map" and models["siglip"].n_tokens == (S // P) ** 2
    d_img = torch.from_numpy(gf.synthetic_images(B, S, seed=2024)).cuda()
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

    for m in models.values():
        window(m, args.warmup)
    rates = {k: [] for k in models}
    for _ in range(args.rounds):
        for k, m in models.items():
            rates[k].append(round(window(m, args.steps), 1))
    med = {k: float(np.median(v)) for k, v in rates.items()}
    prof = {}
    for k, m in models.items():
        check(Lb.vitb200_profile_enable(m.handle, 1))
        for _ in range(args.steps):
            call(m)
        prof[k] = {}
        for i, kind in enumerate(KINDS):
            ms, n, fl = C.c_double(), C.c_int(), C.c_double()
            check(Lb.vitb200_profile_read(m.handle, i, C.byref(ms), C.byref(n), C.byref(fl)))
            prof[k][kind] = {"ms_per_step": round(ms.value / args.steps, 3), "launches_per_step": n.value // args.steps}
        check(Lb.vitb200_profile_enable(m.handle, 0))
        prof[k]["launches"] = m.last_launch_count()
    # the probe-attention kernel alone, from a torch.profiler window of its own
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as tp:
        for _ in range(args.steps):
            call(models["siglip"])
        torch.cuda.synchronize()
    ka = [a for a in tp.key_averages() if "attention_pool_kernel" in a.key]
    n_ap = sum(a.count for a in ka)
    us_mean = sum(a.device_time_total for a in ka) / n_ap if n_ap else None
    NP = (S // P) ** 2
    bound_us = 4.0 * NP * D * B / HBM_BYTES_PER_S * 1e6
    apool = {"launches": n_ap, "us_mean": round(us_mean, 2) if us_mean else None, "hbm_bound_us": round(bound_us, 2),
             "share_of_hbm_bound": round(bound_us / us_mean, 3) if us_mean else None, "bytes": 4 * NP * D * B}
    for m in models.values():
        m.close()
    fc1 = {k: prof[k]["fc1"]["ms_per_step"] for k in prof}
    return {"shape": f"{label} ({L} layers, D {D}; {NP + 1} tokens reference, {NP} SigLIP)", "batch": B, "images_per_s": rates,
            "median_images_per_s": med, "siglip_over_reference": round(med["siglip"] / med["reference"], 4),
            "fc1_ms_activation3_vs_activation0": fc1, "attention_pool_kernel": apool, "profiled": prof}


def main():
    tmp = tempfile.mkdtemp(prefix="bench_siglip_")
    out = {"card": card_info(0), "steps": args.steps, "rounds": args.rounds, "pairs": []}
    for label, (shape, B) in PAIRS.items():
        out["pairs"].append(run_pair(tmp, label, shape, B))
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


main()
