"""Dev tool (run under gpurun): per-image parity distribution of a config against the live reference (oracle/_ref), or against
tests/golden/<cfg>_f16_b64.npz when it exists.  usage: python tools/parity_dist.py <cfg> <ftype> <n_images> [seed] [threads]"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.util import pkg, gf, model_path  # noqa: E402
from oracle import ref  # noqa: E402

eng = pkg.engine
cfg = sys.argv[1] if len(sys.argv) > 1 else "base"
ft = sys.argv[2] if len(sys.argv) > 2 else "f16"
n = int(sys.argv[3]) if len(sys.argv) > 3 else 64
seed = int(sys.argv[4]) if len(sys.argv) > 4 else 777
threads = int(sys.argv[5]) if len(sys.argv) > 5 else min(64, os.cpu_count() or 8)
path = model_path(cfg, ft)
m = eng.vit_model_load(path, 0, max(n, 1))
imgs = gf.synthetic_images(n, m.img_size, seed=seed)
probs, idx, val, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
gold = os.path.join(ROOT, "tests", "golden", f"{cfg}_{ft}_b{n}.npz")
floor = None
if os.path.exists(gold) and int(np.load(gold)["image_seed"]) == seed:
    g = np.load(gold)
    l_ref, p_ref = g["logits"], g["probs"]
    floor = g["floor"] if "floor" in g else None
    src = "golden"
else:
    rm = ref.RefModel(path)
    t = time.time()
    p_ref, l_ref = rm.predict_batch(imgs, n_threads=threads)
    src = "live reference, %d threads, %.1f s" % (threads, time.time() - t)
    rm.close()
re = np.abs(logits - l_ref).max(1) / np.abs(l_ref).max(1)
l2 = np.linalg.norm(logits - l_ref, axis=1) / np.linalg.norm(l_ref, axis=1)
order = np.argsort(-l_ref, 1)[:, :5]
top5 = (order == idx).all(1)
print(f"{cfg} {ft} n={n} vs {src}")
print(f"  max-norm rel: median {np.median(re):.3e} p90 {np.quantile(re, 0.9):.3e} max {re.max():.3e} mean {re.mean():.3e}; images > 1e-3: {(re > 1e-3).sum()}")
print(f"  L2 rel: median {np.median(l2):.3e} max {l2.max():.3e}; top-1 match {(order[:, 0] == idx[:, 0]).mean():.3f}; top-5 lists identical {top5.sum()}/{n}")
if floor is not None:
    print(f"  floor (variant 1): median {np.median(floor):.3e} p90 {np.quantile(floor, 0.9):.3e} max {floor.max():.3e}; ratio of medians {np.median(re) / np.median(floor):.3f}")
m.close()
