"""CPU tests of the kernel test hooks' device check: without a GPU every hook that launches a kernel fails with the engine's
"no CPU fallback" message instead of running on the host or reporting a raw CUDA error.  And the GEMM hooks' epilogue and shape checks,
which come before the device is touched, so they hold on any machine."""
import os
import re

import numpy as np
import pytest

from tests.util import pkg

eng = pkg.engine

M = N = K = 128
D, ROWS = 128, 8
B, NT, H = 1, 16, 1


def _attention_parts(hd, causal=False):
    z = np.zeros((B * NT, 3 * H * hd), np.float16)
    return eng.test_attention_parts(z, z, B, NT, H, hd, causal)


HOOKS = {
    "gemm": lambda: eng.test_gemm(M, N, K, eng.EPI_BIAS_F16, np.zeros((M, K), np.float16), np.zeros((N, K), np.float16), np.zeros(N, np.float32)),
    "gemm_layer_scale": lambda: eng.test_gemm_layer_scale(M, N, K, np.zeros((M, K), np.float16), np.zeros((N, K), np.float16),
                                                          np.zeros(N, np.float32), np.ones(N, np.float32), np.zeros((M, N), np.float32)),
    "gemm_fp8": lambda: eng.test_gemm_fp8(M, N, K, eng.EPI_BIAS_F16, np.zeros((M, K), np.uint8), np.ones(M, np.float32), np.zeros((N, K), np.uint8),
                                          1.0, np.zeros(N, np.float32)),
    "gemm_planes": lambda: eng.test_gemm_planes(M, N, K, eng.EPI_BIAS_F16, np.zeros((M, K), np.float16), np.zeros((N, K), np.float16),
                                                np.zeros(N, np.float32), M),
    "gemm_q8": lambda: eng.test_gemm_q8(np.zeros((M, K), np.float32), np.zeros(N * (K // 32) * 34, np.uint8), np.zeros(N, np.float32)),
    "layernorm": lambda: eng.test_layernorm(np.zeros((ROWS, D), np.float32), np.ones(D, np.float32), np.zeros(D, np.float32)),
    "layernorm_fp8": lambda: eng.test_layernorm_fp8(np.zeros((ROWS, D), np.float32), np.ones(D, np.float32), np.zeros(D, np.float32)),
    "attention": lambda: eng.test_attention(np.zeros((B * NT, 3 * H * 64), np.float16), B, NT, H),
    "attention_hilo": lambda: eng.test_attention_hilo(np.zeros((B * NT, 3 * H * 64), np.float32), B, NT, H),
    "attention_parts": lambda: _attention_parts(64),
    "attention_parts_causal": lambda: _attention_parts(64, causal=True),
    "attention_parts_hd80": lambda: _attention_parts(80),
    "attention_parts_hd72": lambda: _attention_parts(72),
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


def _planes(epi=eng.EPI_BIAS_F16, n=N, k=K, plane_rows=M, e4m3=False):
    dt = np.uint8 if e4m3 else np.float16
    return eng.test_gemm_planes(M, n, k, epi, np.zeros((M, k), dt), np.zeros((n, k), dt), np.zeros(n, np.float32), plane_rows,
                                a_scale=np.ones(M, np.float32) if e4m3 else None)


@pytest.mark.parametrize("epi", [e for e in range(-1, 13) if e not in (eng.EPI_BIAS_F16, eng.EPI_BIAS_F16_HILO)])
def test_gemm_planes_hook_refuses_other_epilogues(epi):
    """Only the qkv and k | v GEMMs write head-major planes: epilogue 0 and the split-precision 6, refused on the host otherwise."""
    with pytest.raises(eng.VitB200Error, match=rf"head-major GEMM epilogue {epi} not supported \(0, 6:"):
        _planes(epi)


@pytest.mark.parametrize("e4m3", [False, True])
def test_gemm_planes_hook_refuses_shapes_it_has_no_map_for(e4m3):
    """A plane is 64 columns wide (N % 64), holds every row (plane_rows >= M), and the operand rows are 16-byte strides (K % 8 for f16,
    K % 16 for e4m3): each refused before the device is touched, naming the limit."""
    kmul = 16 if e4m3 else 8
    with pytest.raises(eng.VitB200Error, match=rf"bad shape \(M >= 1, N a multiple of 64, K a multiple of {kmul}; got M = 128, N = 96,"):
        _planes(n=96, e4m3=e4m3)
    with pytest.raises(eng.VitB200Error, match=rf"K a multiple of {kmul}; got M = 128, N = 128, K = {kmul + 4}\)"):
        _planes(k=kmul + 4, e4m3=e4m3)
    with pytest.raises(eng.VitB200Error, match=r"plane_rows = 127 out of range \(M = 128 \.\. 2\^31 - 1\)"):
        _planes(plane_rows=M - 1, e4m3=e4m3)
    if e4m3:
        with pytest.raises(eng.VitB200Error, match=r"K a multiple of 16; got M = 128, N = 128, K = 40\)"):
            _planes(k=40, e4m3=True)  # a multiple of 8: an f16 row length, not an e4m3 one


def test_gemm_planes_hook_refuses_a_missing_or_stray_lo_buffer():
    """Epilogue 6 writes lo planes: it needs the buffer, and epilogue 0 must not be given one.  An e4m3 run needs its A scales, an f16
    one takes none."""
    L = eng.lib()
    a = np.zeros(M * K, np.float16)
    f = np.zeros(max(M, N), np.float32)
    hi, lo = np.zeros(N * M, np.uint16), np.zeros(N * M, np.uint16)
    for epi, lo_p in ((eng.EPI_BIAS_F16_HILO, None), (eng.EPI_BIAS_F16, lo.ctypes.data)):
        assert L.vitb200_test_gemm_planes(0, M, N, K, epi, M, 0, a.ctypes.data, None, a.ctypes.data, 1.0, f.ctypes.data, hi.ctypes.data,
                                          lo_p) != 0
        assert "lo goes with epilogue 6, and only with it" in eng.lib().vitb200_last_error().decode()
    for e4m3, sa in ((1, None), (0, f.ctypes.data)):
        assert L.vitb200_test_gemm_planes(0, M, N, K, eng.EPI_BIAS_F16, M, e4m3, a.ctypes.data, sa, a.ctypes.data, 1.0, f.ctypes.data,
                                          hi.ctypes.data, None) != 0
        assert "a_scale goes with e4m3 operands, and only with them" in eng.lib().vitb200_last_error().decode()
