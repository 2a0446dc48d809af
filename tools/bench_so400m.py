"""Dev tool (one H100): SigLIP So400m-384's 72-column attention heads against 64-column heads at the same width.
Two seeded synthetic map-pool towers of the same shape -- D 1152, 27 layers, MLP 4304, patch 14, 384 px (a 27 x 27 grid, 729 tokens), the
attention-pooling head -- one with 16 heads of 72 columns (So400m) and one with 18 heads of 64, at batch 64, images resident on the device.
Both do the same attention FLOPs (4 N^2 D per image per layer).  At 729 tokens the head-dim-72 model runs attention_rowmajor_kernel<72>
on f16 operands with 16 warps, the head-dim-64 one the 8-warp attention_kernel (729 > 640).
    1. images/s of vitb200_forward_device over R rounds of K calls, alternating the two models in one process (host clock from a
       synchronised device to a device synchronise);
    2. a separate profiled pass per model (vitb200_profile_*): attention ms per step and TFLOP/s, the pooling head (kind 8) ms per step,
       and the step's other kernel kinds.
The card name, power limit and max SM clock are read in the same run.
usage: python tools/bench_so400m.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
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
D, L, F, P, S = 1152, 27, 4304, 14, 384
CLASSES = D   # the map tower's identity head: its logits are the pooled row
HEADS = {"hd72": 16, "hd64": 18}

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=64)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_so400m.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


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


def synth_tensors(seed=7):
    """Seeded weights of the tower (the same for both head counts): matrices randn / sqrt(fan in), LayerNorms near the identity."""
    rng = np.random.default_rng(seed)
    mat = lambda r, c: (rng.standard_normal((r, c), np.float32) / np.sqrt(c)).astype(np.float16)
    vec = lambda n, s=0.02: (s * rng.standard_normal(n)).astype(np.float32)
    G = S // P
    t = {"pos_embed": vec(G * G * D, 0.5).reshape(1, G * G, D), "patch_embed.proj.weight": mat(D, 3 * P * P).reshape(D, 3, P, P),
         "patch_embed.proj.bias": vec(D).reshape(1, D, 1, 1)}
    for i in range(L):
        b = f"blocks.{i}."
        t.update({b + "norm1.weight": 1 + vec(D, 0.1), b + "norm1.bias": vec(D), b + "attn.qkv.weight": mat(3 * D, D), b + "attn.qkv.bias": vec(3 * D),
                  b + "attn.proj.weight": mat(D, D), b + "attn.proj.bias": vec(D), b + "norm2.weight": 1 + vec(D, 0.1), b + "norm2.bias": vec(D),
                  b + "mlp.fc1.weight": mat(F, D), b + "mlp.fc1.bias": vec(F), b + "mlp.fc2.weight": mat(D, F), b + "mlp.fc2.bias": vec(D)})
    t.update({"norm.weight": 1 + vec(D, 0.1), "norm.bias": vec(D), "head.weight": np.eye(D, dtype=np.float16), "head.bias": vec(D, 0.0),
              "attn_pool.latent": vec(D, 0.5).reshape(1, 1, D), "attn_pool.q.weight": mat(D, D), "attn_pool.q.bias": vec(D),
              "attn_pool.kv.weight": mat(2 * D, D), "attn_pool.kv.bias": vec(2 * D), "attn_pool.proj.weight": mat(D, D),
              "attn_pool.proj.bias": vec(D), "attn_pool.norm.weight": 1 + vec(D, 0.1), "attn_pool.norm.bias": vec(D),
              "attn_pool.mlp.fc1.weight": mat(F, D), "attn_pool.mlp.fc1.bias": vec(F), "attn_pool.mlp.fc2.weight": mat(D, F),
              "attn_pool.mlp.fc2.bias": vec(D)})
    return t


def model_file(directory, heads, tensors):
    """The tower as GGUF (f16 matrices, gelu_pytorch_tanh, pool 'map') with `heads` attention heads."""
    vf = gf.VitFile(D, L, heads, CLASSES, P, S, 1, activation="gelu_pytorch_tanh", pool="map")
    for name, arr in tensors.items():
        vf.tensors[name] = arr
        vf.tensor_ftype[name] = 1 if arr.dtype == np.float16 else 0
    path = os.path.join(directory, f"h{heads}.gguf")
    gf.write_gguf(path, vf)
    return path


def check(rc):
    if rc:
        raise RuntimeError(eng.lib().vitb200_last_error().decode())


def main():
    B = args.batch
    N = (S // P) ** 2
    tmp = tempfile.mkdtemp(prefix="bench_so400m_")
    t = synth_tensors()
    models = {k: eng.vit_model_load(model_file(tmp, h, t), 0, B) for k, h in HEADS.items()}
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

    out = {"card": card_info(0), "shape": f"D {D}, {L} layers, F {F}, {N} tokens, map pool, batch {B}", "steps": args.steps,
           "rounds": args.rounds}
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
    for f in os.listdir(tmp):
        os.remove(os.path.join(tmp, f))
    os.rmdir(tmp)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
