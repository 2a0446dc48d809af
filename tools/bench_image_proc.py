"""Dev tool (one H100): Hugging Face image preprocessing on the GPU (vitb200_set_image_proc) against no preprocessing at all.
Two seeded synthetic towers, GGUF with f16 matrices, batch 256 of seeded random RGB photos, each side uniform in 200..1200 px:
    SigLIP B/16-224 MAP tower (as tools/bench_siglip.py builds it) with SigLIP's processor: bicubic resize to 224 x 224
    B/16-224 tower of the reference architecture with CLIP's processor: bicubic resize of the short side to 224, centre crop 224
For each, R rounds alternate two windows of K blocking calls (host clock, device synchronised at both ends):
    u8    vit_features_u8 on the photos through the processor (pooled rows out): packing, one H2D copy, the two kernels, the encoder
    f32   vit_features on the same photos' pixel_values, prepared beforehand by the PIL processor: the ceiling without preprocessing
A torch.profiler window of its own then gives the device time of image_proc_h_kernel and image_proc_v_kernel per batch.  Also reported:
the host-to-device bytes per batch of both paths, the PIL processor's host time per image in this process (transformers' PIL backend,
one process, measured on up to 64 of the photos), and the card name, power limit and max SM clock, read in the same run.
usage: python tools/bench_image_proc.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
import argparse
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
CLASSES = 1000
SHAPE = (768, 12, 12, 16, 224)  # B/16 at 224
KERNELS = ("image_proc_h_kernel", "image_proc_v_kernel")

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=256)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_image_proc.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


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


def model_file(directory, siglip):
    """A seeded synthetic B/16-224 model (ggml_file.synth_tensors); the SigLIP one drops the class token and its position row and adds
    the 13 attention-pooling head tensors."""
    D, L, H, P, S = SHAPE
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
    path = os.path.join(directory, f"{'siglip' if siglip else 'clip'}-b16-224.gguf")
    gf.write_gguf(path, vf)
    return path


def photos(B, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (int(rng.integers(200, 1201)), int(rng.integers(200, 1201)), 3), dtype=np.uint8) for _ in range(B)]


def run(tmp, label, siglip, proc):
    from PIL import Image
    B, S = args.batch, SHAPE[4]
    m = eng.vit_model_load(model_file(tmp, siglip), 0, B)
    m.set_image_proc(proc.to_dict())
    imgs = photos(B, seed=2026 + siglip)
    pil = [Image.fromarray(a) for a in imgs]
    n_host = min(B, 64)
    t0 = time.perf_counter()
    pv = proc(pil[:n_host], return_tensors="np")["pixel_values"]
    host_ms = (time.perf_counter() - t0) * 1e3 / n_host
    pv = np.ascontiguousarray(np.asarray(proc(pil, return_tensors="np")["pixel_values"], np.float32).transpose(0, 2, 3, 1))
    calls = {"u8": lambda: eng.vit_features_u8(m, imgs, tokens=False, prelogits=True),
             "f32": lambda: eng.vit_features(m, pv, tokens=False, prelogits=True)}
    # the two paths compute the same rows: the u8 path's pixels are the processor's
    assert np.array_equal(calls["u8"]()[1], calls["f32"]()[1])

    def window(call, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            call()
        torch.cuda.synchronize()
        return B * steps / (time.perf_counter() - t0)

    for call in calls.values():
        window(call, args.warmup)
    rates = {k: [] for k in calls}
    for _ in range(args.rounds):
        for k, call in calls.items():
            rates[k].append(round(window(call, args.steps), 1))
    med = {k: float(np.median(v)) for k, v in rates.items()}
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as tp:
        for _ in range(args.steps):
            calls["u8"]()
        torch.cuda.synchronize()
    kern = {}
    for name in KERNELS:
        ka = [a for a in tp.key_averages() if name in a.key]
        n = sum(a.count for a in ka)
        kern[name] = {"launches": n, "us_per_batch": round(sum(a.device_time_total for a in ka) / args.steps, 1)}
    staged = sum((a.size + 255) // 256 * 256 for a in imgs) + B * (16 + 40)  # pixels, PreImage and ProcGeom rows
    m.close()
    return {"model": label, "processor": gf.image_proc_from_config(proc.to_dict(), S), "batch": B,
            "photo_pixels_mean": round(float(np.mean([a.shape[0] * a.shape[1] for a in imgs])), 1),
            "images_per_s": rates, "median_images_per_s": med, "u8_over_f32": round(med["u8"] / med["f32"], 4),
            "preprocess_kernels": kern, "h2d_bytes_per_batch": {"u8": staged, "f32": B * S * S * 3 * 4},
            "pil_host_ms_per_image": round(host_ms, 2)}


def main():
    import transformers as tr
    tmp = tempfile.mkdtemp(prefix="bench_image_proc_")
    out = {"card": card_info(0), "steps": args.steps, "rounds": args.rounds, "runs": []}
    out["runs"].append(run(tmp, "SigLIP B/16-224 MAP tower, 12 layers", True, tr.SiglipImageProcessorPil()))
    out["runs"].append(run(tmp, "B/16-224, 12 layers, reference architecture", False, tr.CLIPImageProcessorPil()))
    print(json.dumps(out), flush=True)


main()
