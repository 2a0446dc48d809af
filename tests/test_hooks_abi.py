"""CPU tests of the kernel test hooks' device check: without a GPU every hook that launches a kernel fails with the engine's
"no CPU fallback" message instead of running on the host or reporting a raw CUDA error.  And the GEMM hook's epilogue check, which
comes before the device is touched, so it holds on any machine."""
import os
import re

import numpy as np
import pytest

from tests.util import pkg

eng = pkg.engine

M = N = K = 128
D, ROWS = 128, 8
B, NT, H = 1, 16, 1

HOOKS = {
    "gemm": lambda: eng.test_gemm(M, N, K, eng.EPI_BIAS_F16, np.zeros((M, K), np.float16), np.zeros((N, K), np.float16), np.zeros(N, np.float32)),
    "gemm_layer_scale": lambda: eng.test_gemm_layer_scale(M, N, K, np.zeros((M, K), np.float16), np.zeros((N, K), np.float16),
                                                          np.zeros(N, np.float32), np.ones(N, np.float32), np.zeros((M, N), np.float32)),
    "gemm_fp8": lambda: eng.test_gemm_fp8(M, N, K, eng.EPI_BIAS_F16, np.zeros((M, K), np.uint8), np.ones(M, np.float32), np.zeros((N, K), np.uint8),
                                          1.0, np.zeros(N, np.float32)),
    "gemm_q8": lambda: eng.test_gemm_q8(np.zeros((M, K), np.float32), np.zeros(N * (K // 32) * 34, np.uint8), np.zeros(N, np.float32)),
    "layernorm": lambda: eng.test_layernorm(np.zeros((ROWS, D), np.float32), np.ones(D, np.float32), np.zeros(D, np.float32)),
    "layernorm_fp8": lambda: eng.test_layernorm_fp8(np.zeros((ROWS, D), np.float32), np.ones(D, np.float32), np.zeros(D, np.float32)),
    "attention": lambda: eng.test_attention(np.zeros((B * NT, 3 * H * 64), np.float16), B, NT, H),
    "attention_hilo": lambda: eng.test_attention_hilo(np.zeros((B * NT, 3 * H * 64), np.float32), B, NT, H),
    "softmax_topk": lambda: eng.test_softmax_topk(np.zeros((ROWS, 10), np.float32), 5),
    "attention_pool": lambda: eng.test_attention_pool(np.zeros(H * 64, np.float32), np.zeros((B * NT, 2 * H * 64), np.float16), B, NT, H),
}


@pytest.mark.parametrize("hook", sorted(HOOKS))
def test_device_hooks_have_no_cpu_fallback(hook):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(eng.VitB200Error) as ei:
        HOOKS[hook]()
    assert "no CPU fallback" in str(ei.value)


def _gemm(epi):
    return eng.test_gemm(M, N, K, epi, np.zeros((M, K), np.float16), np.zeros((N, K), np.float16), np.zeros(N, np.float32),
                         np.zeros((M, N), np.float32))


@pytest.mark.parametrize("epi", [eng.EPI_PATCH_F32, 5, 12, -1, 1 << 20])
def test_gemm_hook_refuses_unlisted_epilogues(epi):
    """Epilogue 3 (the patch embedding) would read a position table the hook does not take, and the rest are no epilogue at all: all
    refused on the host, before the device check, so the message is the same with and without a GPU."""
    with pytest.raises(eng.VitB200Error, match=rf"GEMM epilogue {epi} not supported \(0, 1, 2, 4, 6, 7, 8, 10, 11;"):
        _gemm(epi)


def test_epilogue_ids_match_the_kernel():
    """engine.py's EPI_* names and values are those of enum GemmEpilogue in csrc/gemm_wgmma.cuh, parsed as declared_symbols() parses
    the header."""
    src = open(os.path.join(os.path.dirname(eng.LIB_PATH), "csrc", "gemm_wgmma.cuh")).read()
    body = re.search(r"enum GemmEpilogue\s*\{(.*?)\};", src, re.S).group(1)
    declared = {name: int(value) for name, value in re.findall(r"^\s*(EPI_\w+)\s*=\s*(\d+)\s*,", re.sub(r"//[^\n]*", "", body), re.M)}
    exported = {name: getattr(eng, name) for name in dir(eng) if name.startswith("EPI_") and name != "EPI_SWIGLU"}
    assert exported == declared
    assert eng.EPI_SWIGLU == eng.EPI_BIAS_SWIGLU_F16


def test_gemm_hook_sends_layer_scale_to_its_own_hook():
    with pytest.raises(eng.VitB200Error, match="vitb200_test_gemm_layer_scale"):
        _gemm(eng.EPI_BIAS_SCALE_RESID_F32)
