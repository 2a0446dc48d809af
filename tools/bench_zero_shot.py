"""Dev tool (one H100): zero-shot classification on the GPU (vitb200_set_zero_shot) against the host recipe it replaces, on a seeded
CLIP ViT-B/16-shaped image tower (12 layers, D 768, patch 16, 224 px, pre-norm, QuickGELU, E 512) at batch 256, images resident on the
device, for C = 1000 (ImageNet) and C = 21 843 (ImageNet-21k) classes.  Two paths, alternated over R rounds of K calls in one process (host
clock from a synchronised device to a synchronised device), each ending with the top-5 ids and probabilities on the host:
    gpu   vitb200_forward_device with the head set: top-5 on the device, then the 256 x 5 results copied back
    host  vitb200_forward_device without a head: the 256 x 512 embeddings copied back, zero_shot_logits (float64 numpy), soft-max, top-5
Then one torch.profiler window of the gpu path for the device time of the similarity kernel and the soft-max + top-k kernel.  The card's
name, power limit and maximum SM clock are read in the same run.
usage: python tools/bench_zero_shot.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
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
SHAPE = (768, 12, 12, 16, 224)  # hidden, layers, heads, patch, img
PROJ = 512
CLASSES = (1000, 21843)
LOGIT_SCALE = float(np.log(100.0))

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=256)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_zero_shot.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


def card_info():
    """Name, power limit and maximum SM clock of the GPU the numbers were measured on (read-only query)."""
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30)
    return q.stdout.strip()


def model_file(directory):
    """A seeded CLIP tower (ggml_file.synth_tensors plus norm_pre, QuickGELU, eps 1e-5), GGUF with f16 matrices."""
    D, L, H, P, S = SHAPE
    vf = gf.VitFile(D, L, H, PROJ, P, S, 1)
    for name, arr in gf.synth_tensors(D, L, PROJ, P, S, seed=7).items():
        f16 = arr.ndim >= 2 and name not in ("cls_token", "pos_embed")
        if name == "patch_embed.proj.bias":
            arr = arr.reshape(1, -1, 1, 1)
        vf.tensors[name] = arr.astype(np.float16 if f16 else np.float32)
        vf.tensor_ftype[name] = 1 if f16 else 0
    rng = np.random.default_rng(8)
    vf.tensors["norm_pre.weight"] = (1 + 0.02 * rng.standard_normal(D)).astype(np.float32)
    vf.tensors["norm_pre.bias"] = (0.02 * rng.standard_normal(D)).astype(np.float32)
    vf.tensor_ftype["norm_pre.weight"] = vf.tensor_ftype["norm_pre.bias"] = 0
    vf.pre_norm, vf.activation, vf.eps = 1, "quick_gelu", 1e-5
    path = os.path.join(directory, "clip_b16.gguf")
    gf.write_gguf(path, vf)
    return path


def check(rc):
    if rc:
        raise RuntimeError(eng.lib().vitb200_last_error().decode())


def main():
    B = args.batch
    path = model_file(tempfile.mkdtemp(prefix="bench_zero_shot_"))
    d_img = torch.from_numpy(gf.synthetic_images(B, SHAPE[4], seed=2024)).cuda()
    plain = eng.vit_model_load(path, 0, B)
    d_emb = torch.empty((B, PROJ), dtype=torch.float32, device="cuda")
    print(json.dumps({"gpu": card_info(), "batch": B, "shape": "CLIP ViT-B/16 image tower, E 512"}))
    for n_cls in CLASSES:
        T = np.random.default_rng(n_cls).standard_normal((n_cls, PROJ)).astype(np.float32)
        zs = eng.vit_model_load(path, 0, B)
        zs.set_zero_shot(T, LOGIT_SCALE, probs="softmax")
        d_idx = torch.empty((B, 5), dtype=torch.int32, device="cuda")
        d_val = torch.empty((B, 5), dtype=torch.float32, device="cuda")

        def gpu_step():
            check(eng.lib().vitb200_forward_device(zs.handle, d_img.data_ptr(), B, None, None, d_idx.data_ptr(), d_val.data_ptr(), 5, None))
            check(eng.lib().vitb200_sync(zs.handle))
            return d_idx.cpu().numpy(), d_val.cpu().numpy()

        def host_step():
            check(eng.lib().vitb200_forward_device(plain.handle, d_img.data_ptr(), B, None, d_emb.data_ptr(), None, None, 0, None))
            check(eng.lib().vitb200_sync(plain.handle))
            lg = eng.zero_shot_logits(d_emb.cpu().numpy(), T, LOGIT_SCALE)
            p = np.exp(lg - lg.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            idx = np.argsort(-p, axis=1, kind="stable")[:, :5]
            return idx, np.take_along_axis(p, idx, 1)

        g_idx, _ = gpu_step()
        h_idx, _ = host_step()
        agree = float((g_idx[:, 0] == h_idx[:, 0]).mean())
        rates = {"gpu": [], "host": []}
        for _ in range(args.rounds):
            for name, step in (("gpu", gpu_step), ("host", host_step)):
                for _ in range(args.warmup):
                    step()
                torch.cuda.synchronize()
                t = time.perf_counter()
                for _ in range(args.steps):
                    step()
                torch.cuda.synchronize()
                rates[name].append(B * args.steps / (time.perf_counter() - t))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                gpu_step()
            torch.cuda.synchronize()
        dev = {"zero_shot_kernel": 0.0, "softmax_topk_kernel": 0.0}
        for ev in prof.key_averages():
            for k in dev:
                if k in ev.key:
                    dev[k] += ev.device_time_total / 1e3 / args.steps  # ms per forward
        flops = 2.0 * B * n_cls * PROJ
        print(json.dumps({"classes": n_cls, "images_per_s": {k: [round(x, 1) for x in v] for k, v in rates.items()},
                          "top1_agreement_gpu_vs_host": agree, "device_ms_per_forward": {k: round(v, 4) for k, v in dev.items()},
                          "similarity_tflops": round(flops / (dev["zero_shot_kernel"] * 1e-3) / 1e12, 2) if dev["zero_shot_kernel"] else None}))
        zs.close()
    plain.close()


if __name__ == "__main__":
    main()
