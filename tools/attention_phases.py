"""Dev tool (needs an H100): where a split-precision attention CTA's time goes, from the kernels' phase probe
(vitb200_test_attention_phases, csrc/attention_wgmma.cuh), at the bench shape (ViT-B/16: 12 heads, 197 tokens, batch 256).

For the one-CTA-per-(image, head) kernel and the persistent kernel, the medians over every recorded problem and computing warpgroup of
  wait     its first q tile's operands: from the moment it asks for them to the moment they have landed
  S        S = Q K^T of that tile (three products per k16 step)
  softmax+PV   the soft-max and O = P V of that tile
and for the per-head kernel the load latency (K V issued -> landed), with the launch's span from the first stamp to the last.

    python tools/attention_phases.py [--batch 256] [--tokens 197]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.util import pkg  # noqa: E402

eng = pkg.engine


def phases(rec):
    """rec [grid, problems, fields] -> dict of medians (us) and the span (us)"""
    issued = rec[:, :, 0].astype(np.int64)
    out = {"wait": [], "S": [], "softmax+PV": [], "load": []}
    for c in range(2):
        f = rec[:, :, 1 + 4 * c: 5 + 4 * c].astype(np.int64)
        ok = (f > 0).all(axis=2)
        out["wait"] += list((f[..., 1] - f[..., 0])[ok])
        out["S"] += list((f[..., 2] - f[..., 1])[ok])
        out["softmax+PV"] += list((f[..., 3] - f[..., 2])[ok])
        out["load"] += list((f[..., 1] - issued)[ok & (issued > 0)])
    stamps = rec[rec > 0].astype(np.int64)
    med = {k: float(np.median(v)) / 1e3 for k, v in out.items() if v}
    return med, (stamps.max() - stamps.min()) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--tokens", type=int, default=197)
    ap.add_argument("--heads", type=int, default=12)
    a = ap.parse_args()
    B, N, H = a.batch, a.tokens, a.heads
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}; B = {B}, N = {N}, H = {H}: {B * H} problems")
    qkv = np.random.default_rng(0).standard_normal((B * N, 3 * H * 64)).astype(np.float32)
    for name, kernel in (("per (image, head) CTA", eng.ATTN_WGMMA_HEAD), ("persistent", eng.ATTN_WGMMA)):
        eng.test_attention_phases(qkv, B, N, H, kernel)  # warm-up: module load, shared-memory opt-in
        rec = eng.test_attention_phases(qkv, B, N, H, kernel)
        med, span = phases(rec)
        grid = rec.shape[0]
        print(f"{name:22s} grid {grid:5d}: span {span:8.1f} us; per tile (median): " +
              ", ".join(f"{k} {v:.2f} us" for k, v in med.items()))


if __name__ == "__main__":
    main()
