"""Dev tool (GPU): throughput of the q8_0 integer tensor-core GEMM prototype (csrc/gemm_q8_wgmma.cuh) at the ViT-B/16 batch-256
layer shapes, CUDA-event timed inside vitb200_test_gemm_q8.  usage: python tools/bench_q8.py [iters]"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.util import pkg  # noqa: E402

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
M = 256 * 197
rng = np.random.default_rng(0)
rows = []
for name, N, K in (("qkv", 2304, 768), ("proj", 768, 768), ("fc1", 3072, 768), ("fc2", 768, 3072)):
    x = rng.standard_normal((M, K), dtype=np.float32)
    w = (rng.standard_normal((N, K), dtype=np.float32) * 0.05)
    wb = pkg.convert.quantize_q8_0_reference(w.reshape(-1))
    bias = rng.standard_normal(N).astype(np.float32)
    _, _, _, ms = pkg.engine.test_gemm_q8(x, wb, bias, iters=iters)
    ops = 2.0 * M * N * K
    rows.append({"layer": name, "M": M, "N": N, "K": K, "ms_per_launch": ms, "tops": ops / ms / 1e9})
    print(json.dumps(rows[-1]), flush=True)
