"""Text towers (vitb200_create_text) on one GPU: per-call latency at batch 1 (graph replay) and sequences/s at batch 512, for CLIP ViT-L/14's
text tower (12 layers, D 768, 77 tokens, causal), OpenCLIP bigG's (32 layers, D 1280, 20 heads, 77 tokens, causal) and a SigLIP-B-sized
text tower (12 layers, D 768, 64 tokens, bidirectional), on seeded weights; alternated with transformers' CLIPTextModelWithProjection in
float16 on the same GPU and the same ids.  Per-kernel times come from vitb200_profile_*, including the causal attention kernel against the
non-causal one at the same shape.  Prints the card, its power limit and its max SM clock first.

    python tools/bench_text.py [--iters 20]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.util import pkg  # noqa: E402

eng, gf = pkg.engine, pkg.ggml_file

# name: (layers, hidden, heads, context, causal, vocab, projection)
SHAPES = {"clip_l14_text": (12, 768, 12, 77, 1, 49408, 768), "openclip_bigG_text": (32, 1280, 20, 77, 1, 49408, 1280),
          "siglip_b_text": (12, 768, 12, 64, 0, 32000, 768), "clip_l14_text_noncausal": (12, 768, 12, 77, 0, 49408, 768)}


def seeded_file(name, L, D, H, N, causal, V, E):
    rng = np.random.default_rng(0)
    vf = gf.VitFile(D, L, H, E, 0, 0, 1, eps=1e-5, activation="quick_gelu" if causal else "gelu_pytorch_tanh",
                    text={"context": N, "causal": causal, "pool": "eos_argmax" if causal else "last", "eos_token_id": 2,
                          "logit_scale": None, "logit_bias": None})
    def put(k, a, f16):
        vf.tensors[k] = a.astype(np.float16 if f16 else np.float32)
        vf.tensor_ftype[k] = 1 if f16 else 0
    put("token_embd.weight", rng.standard_normal((V, D)) * 0.02, True)
    put("pos_embed", rng.standard_normal((1, N, D)) * 0.01, False)
    for i in range(L):
        p = f"blocks.{i}."
        for k, shape in (("norm1", None), ("attn.qkv", (3 * D, D)), ("attn.proj", (D, D)), ("norm2", None), ("mlp.fc1", (4 * D, D)),
                         ("mlp.fc2", (D, 4 * D))):
            if shape is None:
                put(p + k + ".weight", 1 + 0.02 * rng.standard_normal(D), False)
                put(p + k + ".bias", 0.02 * rng.standard_normal(D), False)
            else:
                put(p + k + ".weight", rng.standard_normal(shape) / np.sqrt(shape[1]), True)
                put(p + k + ".bias", 0.02 * rng.standard_normal(shape[0]), False)
    put("norm.weight", np.ones(D), False)
    put("norm.bias", np.zeros(D), False)
    put("head.weight", rng.standard_normal((E, D)) / np.sqrt(D), True)
    put("head.bias", np.zeros(E), False)
    return vf


def timed(fn, iters):
    import torch
    fn(); fn(); fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", q.stdout.strip())
    for name, (L, D, H, N, causal, V, E) in SHAPES.items():
        vf = seeded_file(name, L, D, H, N, causal, V, E)
        m = eng.vit_model_from_tensors(vf, max_batch=512)
        rng = np.random.default_rng(1)
        for B in (1, 512):
            ids = rng.integers(3, V - 1, (B, N)).astype(np.int32)
            ids[:, N // 2] = V - 1
            d_ids = torch.from_numpy(ids).cuda()
            d_emb = torch.empty((B, E), dtype=torch.float32, device="cuda")
            stream = torch.cuda.current_stream().cuda_stream
            call = lambda: eng._check(eng.lib().vitb200_encode_text_device(m.handle, d_ids.data_ptr(), B, d_emb.data_ptr(), None, None, stream), "enc")
            t = timed(call, a.iters)
            row = f"{name:26s} B={B:4d}  engine {t * 1e3:8.3f} ms/call  {B / t:10.0f} seq/s"
            if causal and E == D or name == "clip_l14_text":
                import transformers as tr
                cfg = tr.CLIPTextConfig(vocab_size=V, hidden_size=D, intermediate_size=4 * D, num_attention_heads=H, num_hidden_layers=L,
                                        max_position_embeddings=N, projection_dim=E)
                hf = tr.CLIPTextModelWithProjection(cfg).half().cuda().eval()
                d64 = d_ids.long()
                with torch.no_grad():
                    th = timed(lambda: hf(input_ids=d64), a.iters)
                row += f"   transformers f16 {th * 1e3:8.3f} ms/call  {B / th:10.0f} seq/s"
                del hf
            print(row, flush=True)
            if B == 512:
                eng._check(eng.lib().vitb200_profile_enable(m.handle, 1), "profile")
                call()
                for kind, kname in ((0, "token gather"), (1, "qkv"), (2, "proj"), (3, "fc1"), (4, "fc2"), (5, "head"), (6, "attention"), (7, "layernorm")):
                    ms, n, fl = C.c_double(), C.c_int(), C.c_double()
                    eng._check(eng.lib().vitb200_profile_read(m.handle, kind, C.byref(ms), C.byref(n), C.byref(fl)), "read")
                    print(f"    {kname:12s} {ms.value:8.3f} ms over {n.value:3d} launches", flush=True)
                eng._check(eng.lib().vitb200_profile_enable(m.handle, 0), "profile")
        m.close()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
