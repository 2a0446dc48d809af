"""Dev tool (one H100): images/s of the encoder-features entry point (`vitb200_features_device`) next to the classification step on
the same ViT-B/16 f16 model, batch, inputs and stream.  Two features workloads:
  prelogits_f32      the pooled, final-LayerNorm'd pre-logits rows at full depth, f32 (the retrieval / linear-probe embedding);
  tokens_f16_penult  every token after block L-1, no LayerNorm, f16 (a multimodal model's vision tower: one block less).
The three workloads are timed in K-step windows (CUDA events on the launching stream), alternated over several rounds so that clock
and neighbour drift hit all of them alike.  The card name and power limit are read in the same run and printed with the rates.
usage: python tools/bench_features.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
# the tree may be read-only: generated model files go to a per-user temporary cache
os.environ.setdefault("VITB200_CACHE", os.path.join(tempfile.gettempdir(), "vitb200-cache-%d" % os.getuid()))
from tests.util import gf, model_path, pkg  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=256)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_features.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


def card_info(index):
    """Name and power limit of the GPU the numbers were measured on (read-only queries)."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


eng = pkg.engine
L = eng.lib()
B = args.batch
model = eng.vit_model_load(model_path("base", "f16"), device=0, max_batch=B)
depth, D = model.hparams.num_hidden_layers, model.hidden_size
# two distinct input batches (2 x 154 MB > 50 MB L2), alternated so no step finds its input in L2
dev_imgs = [torch.from_numpy(gf.synthetic_images(B, model.img_size, seed=1234 + j)).cuda() for j in range(2)]
d_probs = torch.empty(B, model.num_classes, device="cuda")
d_idx = torch.empty(B, 5, dtype=torch.int32, device="cuda")
d_val = torch.empty(B, 5, device="cuda")
d_pre = torch.empty(B, model.head_tokens, D, device="cuda")
d_tok = torch.empty(B, model.n_tokens, D, dtype=torch.float16, device="cuda")
tstream = torch.cuda.Stream()
torch.cuda.set_stream(tstream)
stream = tstream.cuda_stream


def check(rc):
    if rc != 0:
        raise RuntimeError(L.vitb200_last_error().decode())


def classify(i):
    check(L.vitb200_forward_device(model.handle, dev_imgs[i & 1].data_ptr(), B, d_probs.data_ptr(), None, d_idx.data_ptr(),
                                   d_val.data_ptr(), 5, stream))


def features(req, tok, pre):
    def step(i):
        check(L.vitb200_features_device(model.handle, dev_imgs[i & 1].data_ptr(), B, C.byref(req), tok, pre, stream))
    return step


work = {"classification": classify,
        "prelogits_f32": features(eng.FeaturesReq(depth, 1, 0), None, d_pre.data_ptr()),
        "tokens_f16_penult": features(eng.FeaturesReq(depth - 1, 0, 1), d_tok.data_ptr(), None)}
launches = {}
for name, fn in work.items():
    for i in range(args.warmup):
        fn(i)
    torch.cuda.synchronize()
    launches[name] = model.last_launch_count()
ms = {name: 0.0 for name in work}
for _ in range(args.rounds):
    for name, fn in work.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        ms[name] += e0.elapsed_time(e1)
n = args.rounds * args.steps
print(json.dumps({"metric": "images/sec ViT-B/16 224^2, classification vs encoder features", "card": card_info(0), "batch": B,
                  "steps": n, "timing": "%d rounds of %d steps per workload, alternated" % (args.rounds, args.steps),
                  "workloads": {name: {"images_per_s": B * n / (ms[name] * 1e-3), "ms_per_step": ms[name] / n,
                                       "gpu_launches_per_step": launches[name]} for name in work},
                  "output_bytes_per_step": {"prelogits_f32": d_pre.numel() * 4, "tokens_f16_penult": d_tok.numel() * 2}}), flush=True)
model.close()
