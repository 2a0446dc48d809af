"""Dev tool (one H100): images/s of ViTSTR text recognition from u8 word crops (`vitb200_recognize_u8_async`: pinned staging of the u8
images, one upload, grayscale preprocess, forward, greedy decode on the device, ids / lengths / scores back) next to the f32 path it
replaces (`vitb200_forward_async` on the same images already pre-processed to float32 [S][S] in pinned host memory: the 200 KB per
image upload, the forward and the probabilities + top-1 of every token back for a host decode; the host preprocess and the host decode
themselves are not timed, so the f32 rate is an upper bound for that path).
Synthetic ViTSTR-tiny f16 model (D = 192, 12 blocks, 224^2, patch 16), seeded word crops of random size (64-400 x 24-128 pixels).
Each window is K calls timed on the host clock from a synchronised pipeline to vitb200_sync(); the two workloads alternate over
several rounds so that clock and neighbour drift hit both alike.  Where the compiled extension is present (oracle/_ref), the time
of its own scalar preprocess of the same crops on one host thread is reported too.  The card name and power limit are read in the
same run.
usage: python tools/bench_recognize.py [--steps K] [--warmup W] [--rounds R] [--batch B]"""
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
from tests import vitstr_reference as vr  # noqa: E402
from tests.util import model_path, pkg  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=256)
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_recognize.py: no CUDA device; the vit.cpp_b200 forward path has no CPU fallback")


def nvml_power_limit_w(index):
    """The enforced power limit through NVML (read-only), the device found by its PCI address."""
    p = torch.cuda.get_device_properties(index)
    bus = "%08x:%02x:%02x.0" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
    nvml = C.CDLL("libnvidia-ml.so.1")
    if nvml.nvmlInit_v2() != 0:
        return None
    try:
        h, mw = C.c_void_p(), C.c_uint()
        if nvml.nvmlDeviceGetHandleByPciBusId_v2(bus.encode(), C.byref(h)) != 0 or nvml.nvmlDeviceGetEnforcedPowerLimit(h, C.byref(mw)) != 0:
            return None
        return mw.value / 1000.0
    finally:
        nvml.nvmlShutdown()


def card_info(index):
    """Name and power limit of the GPU the numbers were measured on (read-only queries): nvidia-smi, else NVML."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        try:
            info["power_limit_w"] = nvml_power_limit_w(index)
        except Exception as ex:
            info["power_limit_error"] = repr(ex)
    return info


eng = pkg.engine
L = eng.lib()
B = args.batch
model = eng.vit_model_load(model_path("vitstr_tiny", "f16"), device=0, max_batch=B, head_tokens=25)
S, n, NC = model.img_size, model.head_tokens, model.num_classes
rng = np.random.default_rng(1234)
crops = [rng.integers(0, 256, size=(int(rng.integers(24, 129)), int(rng.integers(64, 401)), 3), dtype=np.uint8) for _ in range(B)]
ptrs = (C.c_void_p * B)(*[a.ctypes.data for a in crops])
nx = (C.c_int * B)(*[a.shape[1] for a in crops])
ny = (C.c_int * B)(*[a.shape[0] for a in crops])
u8_bytes = sum(a.nbytes for a in crops)


def pinned(shape, dtype):
    return torch.empty(shape, dtype=dtype).pin_memory()


# f32 path inputs: the same crops pre-processed (bit-identical to the extension's preprocess), in pinned memory
f32 = pinned((B, S, S), torch.float32)
f32.numpy()[:] = eng.vitstr_preprocess_u8(model, crops)
# two output sets per path (one per pipeline slot)
rec_out = [(pinned((B, n - 1), torch.int32), pinned((B,), torch.int32), pinned((B,), torch.float64)) for _ in range(2)]
fwd_out = [(pinned((B, n, NC), torch.float32), pinned((B, n, 1), torch.int32), pinned((B, n, 1), torch.float32)) for _ in range(2)]


def check(rc):
    if rc != 0:
        raise RuntimeError(L.vitb200_last_error().decode())


def recognize(i):
    c, l, s = rec_out[i & 1]
    check(L.vitb200_recognize_u8_async(model.handle, ptrs, nx, ny, B, c.data_ptr(), l.data_ptr(), s.data_ptr(), None))


def forward_f32(i):
    p, ix, v = fwd_out[i & 1]
    check(L.vitb200_forward_async(model.handle, f32.data_ptr(), B, p.data_ptr(), None, ix.data_ptr(), v.data_ptr(), 1))


work = {"recognize_u8": recognize, "forward_f32": forward_f32}
launches = {}
for name, fn in work.items():
    for i in range(args.warmup):
        fn(i)
    check(L.vitb200_sync(model.handle))
    launches[name] = model.last_launch_count()
ms = {name: 0.0 for name in work}
for _ in range(args.rounds):
    for name, fn in work.items():
        check(L.vitb200_sync(model.handle))
        t0 = time.perf_counter()
        for i in range(args.steps):
            fn(i)
        check(L.vitb200_sync(model.handle))
        ms[name] += (time.perf_counter() - t0) * 1e3
# the decode of the last recognition step agrees with the top-1 ids of the f32 path on the same images (same probabilities)
top1 = fwd_out[(args.steps - 1) & 1][1].numpy()[:, 1:, 0]
chars, lengths = rec_out[(args.steps - 1) & 1][0].numpy(), rec_out[(args.steps - 1) & 1][1].numpy()
agree = all(np.array_equal(chars[b, :lengths[b]], top1[b, :lengths[b]]) for b in range(B))
host_pre = None
if vr.available():
    # what the f32 path leaves out: the extension's own scalar preprocess of the same crops, on one host thread
    t0 = time.perf_counter()
    for a in crops:
        vr.preprocess(a, S)
    dt = time.perf_counter() - t0
    host_pre = {"ms_per_step": dt * 1e3, "images_per_s_one_thread": B / dt}
steps = args.rounds * args.steps
print(json.dumps({"metric": "images/sec ViTSTR-tiny 224^2 f16, u8 word crops -> decoded ids vs pre-processed f32 -> probabilities",
                  "card": card_info(0), "batch": B, "steps": steps,
                  "timing": "%d rounds of %d pipelined calls per workload, alternated, host clock to vitb200_sync" % (args.rounds, args.steps),
                  "workloads": {name: {"images_per_s": B * steps / (ms[name] * 1e-3), "ms_per_step": ms[name] / steps,
                                       "gpu_launches_per_step": launches[name]} for name in work},
                  "upload_bytes_per_step": {"recognize_u8": u8_bytes, "forward_f32": B * S * S * 4},
                  "decode_matches_f32_top1": bool(agree), "extension_host_preprocess": host_pre}), flush=True)
model.close()
