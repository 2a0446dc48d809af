"""CPU tests of the drop-in boundary: the C-ABI library loads without a GPU, exports every symbol include/vitb200.h
declares, and fails loudly (no CPU fallback) when asked to compute without a device."""
import os

import numpy as np
import pytest

from tests.util import pkg, gf, model_path

eng = pkg.engine


def test_library_exports_every_declared_symbol():
    L = eng.lib()
    names = eng.declared_symbols()
    assert "vitb200_forward" in names and "vitb200_create_from_file" in names and len(names) >= 12
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing


def test_header_cites_reference_lines():
    src = open(eng.HEADER_PATH).read()
    for cite in ("vit.h:120", "vit.h:122", "vit.cpp:1004-1075", "vit.cpp:308-712"):
        assert cite in src


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(eng.VitB200Error) as ei:
        eng.vit_model_load(model_path("micro", "f16"))
    assert "no CPU fallback" in str(ei.value)


def test_loader_rejects_bad_files(tmp_path):
    import torch
    bad = tmp_path / "bad.gguf"
    bad.write_bytes(b"GGJT" + b"\0" * 64)  # neither the legacy "ggml" magic (vit.cpp:320-328) nor a GGUF container
    with pytest.raises(eng.VitB200Error) as ei:
        eng.vit_model_load(str(bad))
    assert "bad magic" in str(ei.value) or "no CUDA device" in str(ei.value)
    bad.write_bytes(b"GGUF" + b"\0" * 64)  # GGUF magic, garbage behind it: rejected by the container parser (host side, no GPU needed)
    with pytest.raises(eng.VitB200Error) as ei:
        eng.vit_model_load(str(bad))
    assert "invalid GGUF" in str(ei.value)
    with pytest.raises(eng.VitB200Error):
        eng.vit_model_load(str(tmp_path / "missing.gguf"))


def test_product_path_does_not_import_the_oracle():
    """The shipped path (package + csrc) must never route through oracle/."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for dirpath, _, files in os.walk(os.path.join(root, "vit.cpp_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in txt.replace("oracle/vit_oracle.c vo_taps", ""), f"{f} mentions the oracle"


def test_gguf_container_is_parsed_on_the_host(tmp_path):
    """A well-formed GGUF file gets through the container parser (hyper-parameters, tensor inventory, alignment) and only then
    fails for the lack of a GPU; a truncated one is rejected by the parser itself."""
    import torch
    from tests.util import gf
    vf = gf.read(model_path("micro", "f16"))
    good = tmp_path / "micro.gguf"
    gf.write_gguf(str(good), vf, "bf16")
    raw = good.read_bytes()
    assert raw[:4] == b"GGUF"
    if not torch.cuda.is_available():
        with pytest.raises(eng.VitB200Error) as ei:
            eng.vit_model_load(str(good))
        assert "no CUDA device" in str(ei.value)
    cut = tmp_path / "cut.gguf"
    cut.write_bytes(raw[: len(raw) // 2])
    with pytest.raises(eng.VitB200Error) as ei:
        eng.vit_model_load(str(cut))
    assert "invalid GGUF" in str(ei.value) and "wrong size" in str(ei.value)


def test_model_file_parsers_survive_corruption(tmp_path):
    """Truncations and byte flips of valid GGUF and legacy files must come back as errors (or parse and then stop at the
    missing GPU), never crash the process: both loaders are bounds-checked host code."""
    import torch
    from tests.util import gf
    rng = np.random.default_rng(5)
    vf = gf.read(model_path("micro", "f16"))
    good = tmp_path / "m.gguf"
    gf.write_gguf(str(good), vf, "keep")
    for src in (good.read_bytes(), open(model_path("micro", "f16"), "rb").read()):
        head = 4096  # hyper-parameters, labels / metadata and the first tensor records live here
        for trial in range(60):
            raw = bytearray(src)
            if trial % 2 == 0:
                raw = raw[: int(rng.integers(0, len(raw)))]
            else:
                for _ in range(4):
                    raw[int(rng.integers(0, min(head, len(raw))))] = int(rng.integers(0, 256))
            f = tmp_path / f"c{trial}.bin"
            f.write_bytes(bytes(raw))
            try:
                m = eng.vit_model_load(str(f), 0, 2)
                m.close()            # a flip that left the file valid (only possible with a GPU present)
                assert torch.cuda.is_available()
            except eng.VitB200Error:
                pass
            f.unlink()


def test_gguf_parser_under_address_and_ub_sanitizers(tmp_path):
    """csrc/gguf_file.hpp is plain host C++: compile it with -fsanitize=address,undefined and throw 4000 truncated / corrupted
    files at it (tests/cpp/gguf_fuzz.cpp)."""
    import shutil
    import subprocess
    from tests.util import gf
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("no g++")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "gguf_fuzz")
    r = subprocess.run([gxx, "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-I", os.path.join(root, "vit.cpp_b200", "csrc"), os.path.join(root, "tests", "cpp", "gguf_fuzz.cpp"), "-o", exe],
                       capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr.lower():
        pytest.skip("sanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    good = str(tmp_path / "m.gguf")
    gf.write_gguf(good, gf.read(model_path("micro", "f16")), "bf16")
    r = subprocess.run([exe, good, model_path("micro", "f16")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert r.stdout.count("rejected") == 2   # both parsers ran


def test_zeroed_hyper_parameters_are_rejected_not_divided_by(tmp_path):
    """A legacy file whose header says 0 attention heads (or other nonsense) must come back as an error before anything divides
    by it -- checked ahead of the device probe, so it is testable here."""
    import struct
    raw = bytearray(open(model_path("micro", "f16"), "rb").read())
    for field, value in ((3, 0), (1, 0), (5, 0), (2, -7), (6, 1 << 28)):   # heads, hidden, patch, layers, img (header int32 index)
        bad = bytearray(raw)
        struct.pack_into("<i", bad, 4 * field, value)
        f = tmp_path / f"bad{field}.bin"
        f.write_bytes(bytes(bad))
        with pytest.raises(eng.VitB200Error) as ei:
            eng.vit_model_load(str(f))
        assert "invalid" in str(ei.value) or "expected" in str(ei.value), str(ei.value)


@pytest.mark.parametrize("hp,in_chans,limit", [
    ((64, 1, 1, 12, 24), 3, "patch size 12 not supported for 3-channel input (8, 14, 16, 32)"),
    ((64, 1, 1, 14, 28), 1, "patch size 14 not supported for 1-channel input (8, 16)"),
    ((64, 1, 1, 8, 240), 3, "901 tokens not supported (max 896"),
    ((2112, 1, 33, 16, 32), 3, "hidden size 2112 not supported (max 2048)"),
], ids=["patch12", "gray_patch14", "tokens901", "hidden2112"])
def test_shapes_without_a_kernel_are_rejected_at_load(hp, in_chans, limit, tmp_path):
    """Real checkpoints reach these shapes (a grayscale P 14 model, ViT-S/8 at 240 px, a hidden size past the widest LayerNorm): such a
    file must fail to load, naming the limit, instead of loading and then failing in every forward call.  Checked ahead of the device
    probe, so it is testable here; the largest accepted shapes load and run in tests/test_gpu_geometry.py (d2048, p8 at 785 tokens)."""
    f = str(tmp_path / "m.bin")
    gf.write_synthetic(f, hp, 1, classes=10, in_chans=in_chans)
    for fp8 in (False, True):
        with pytest.raises(eng.VitB200Error) as ei:
            eng.vit_model_load(f, fp8=fp8)
        assert limit in str(ei.value), str(ei.value)
