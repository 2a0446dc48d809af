"""Zero-shot heads (vitb200_set_zero_shot) on the CPU: the new symbols are declared and exported, the ctypes mirror of vitb200_zero_shot has
the header's layout, the similarity kernel and the sigmoid top-k compile for sm_90a without spills, and the Python setter refuses a bad
mode or shape before it reaches the engine."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests.util import pkg

eng = pkg.engine
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbols_are_declared_and_exported():
    names = {"vitb200_set_zero_shot", "vitb200_get_zero_shot", "vitb200_num_outputs", "vitb200_test_zero_shot"}
    assert names <= set(eng.declared_symbols())
    L = eng.lib()
    assert all(hasattr(L, n) for n in names)


def test_struct_layout_matches_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if not cc:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vitb200.h"\nint main(void) {\n'
                   'printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(vitb200_zero_shot), offsetof(vitb200_zero_shot, class_embeds), '
                   'offsetof(vitb200_zero_shot, n_classes), offsetof(vitb200_zero_shot, logit_scale), '
                   'offsetof(vitb200_zero_shot, logit_bias), offsetof(vitb200_zero_shot, mode));\nreturn 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    Z = eng.ZeroShot
    assert got == [C.sizeof(Z), Z.class_embeds.offset, Z.n_classes.offset, Z.logit_scale.offset, Z.logit_bias.offset, Z.mode.offset]


def test_kernels_build_for_sm90a_without_spills(tmp_path):
    """The similarity kernel and both forms of the soft-max + top-k kernel through nvcc -Xptxas -v for sm_90a: no spills."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = tmp_path / "k.cu"
    src.write_text('#include "kernels.cuh"\n'
                   "template __global__ void vitb200::softmax_topk_kernel<false>(const float *, int, float *, int32_t *, float *, int, int, float *);\n"
                   "template __global__ void vitb200::softmax_topk_kernel<true>(const float *, int, float *, int32_t *, float *, int, int, float *);\n")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", "-I",
                        os.path.join(ROOT, "vit.cpp_b200", "csrc"), str(src), "-o", str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    info = {}
    for m in re.finditer(r"Compiling entry function '(\w*(?:softmax_topk_kernelILb[01]|zero_shot_kernel)\w*)'.*?"
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr, re.S):
        info[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    assert len(info) == 3, r.stderr
    assert set(info.values()) == {(0, 0)}, info


def test_python_setter_refuses_before_the_engine():
    m = eng.VitModel.__new__(eng.VitModel)  # no engine behind it: these refusals come first
    m._h, m.num_classes = None, 8
    with pytest.raises(ValueError, match="probs must be one of"):
        m.set_zero_shot(np.ones((3, 8), np.float32), 1.0, probs="tanh")
    with pytest.raises(ValueError, match=r"class_embeds must be \[classes, 8\], not \[3, 7\]"):
        m.set_zero_shot(np.ones((3, 7), np.float32), 1.0)
    with pytest.raises(ValueError, match="2 labels for 3 classes"):
        m.set_zero_shot(np.ones((3, 8), np.float32), 1.0, labels=["a", "b"])
    with pytest.raises(ValueError, match="logit_scale is required"):
        m.set_zero_shot(np.ones((3, 8), np.float32))
