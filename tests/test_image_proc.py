"""Hugging Face image processors (vitb200_image_proc) on the CPU: preprocessor_config.json -> the vit.image_proc.* GGUF keys through
the converter and back, every refusal of the config mapping and of the loader (which checks a file's processor before it touches the
device), the GGUF parser fuzzed with a file that carries the keys, and the two kernels compiled for sm_90a without spills."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests.util import pkg, gf, model_path

eng = pkg.engine
cv = pkg.convert
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IMAGENET_MEAN, IMAGENET_STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def _processors():
    """(name, preprocessor config dict) for the three PIL-backend processors' to_dict() and a DINOv2 config (256, then a 224 crop)."""
    import transformers as tr
    return [("clip", tr.CLIPImageProcessorPil().to_dict()), ("siglip", tr.SiglipImageProcessorPil().to_dict()),
            ("bit", tr.BitImageProcessorPil().to_dict()),
            ("dinov2", {"do_resize": True, "size": {"shortest_edge": 256}, "resample": 3, "do_center_crop": True,
                        "crop_size": {"height": 224, "width": 224}, "do_rescale": True, "rescale_factor": 1 / 255, "do_normalize": True,
                        "image_mean": IMAGENET_MEAN, "image_std": IMAGENET_STD})]


def _write_json(path, d):
    with open(path, "w") as f:
        json.dump(d, f, default=int)  # PIL's Resampling is an IntEnum
    return str(path)


def _model_224(tmp_path):
    """A 1-layer RGB model at 224 in the reference's legacy format."""
    path = str(tmp_path / "m224.bin")
    gf.write_synthetic(path, (64, 1, 1, 16, 224), 1, classes=10)
    return path


def _expected(cfg, S=224):
    d = gf.image_proc_from_config(cfg, S)
    d["mean"] = [float(np.float32(x)) for x in d["mean"]]
    d["std"] = [float(np.float32(x)) for x in d["std"]]
    return d


@pytest.mark.parametrize("name", ["clip", "siglip", "bit", "dinov2"])
def test_converter_writes_the_processor_keys(name, tmp_path):
    """convert.py --hf-preprocessor on a converted legacy file: read_gguf returns the keys unchanged (mean and std as float32)."""
    cfg = dict(_processors())[name]
    src, dst = _model_224(tmp_path), str(tmp_path / "out.gguf")
    cv.main([src, dst, "--hf-preprocessor", _write_json(tmp_path / "preprocessor_config.json", cfg)])
    vf = gf.read_gguf(dst)
    assert vf.image_proc == _expected(cfg)
    se = {"clip": 224, "siglip": 0, "bit": 224, "dinov2": 256}[name]
    assert (vf.image_proc["shortest_edge"], vf.image_proc["resample"]) == (se, 3)
    assert (vf.image_proc["crop_height"], vf.image_proc["crop_width"]) == ((0, 0) if name == "siglip" else (224, 224))
    ref = gf.read(src)
    assert set(vf.tensors) == set(ref.tensors)
    assert all(np.array_equal(np.asarray(vf.tensors[k], np.float32), np.asarray(ref.tensors[k], np.float32)) for k in ref.tensors)


def test_converter_writes_the_keys_from_a_hugging_face_checkpoint(tmp_path):
    """The Hugging Face path (a SigLIP tower) carries the processor too; without --hf-preprocessor the file has no keys."""
    import transformers as tr
    from tests import siglip_oracle as so
    m = so.build_hf("micro")
    m.save_pretrained(str(tmp_path))
    cfg = tr.SiglipImageProcessorPil(size={"height": 64, "width": 64}).to_dict()
    args = [str(tmp_path / "model.safetensors"), str(tmp_path / "a.gguf"), "--hf-config", str(tmp_path / "config.json")]
    cv.main(args + ["--hf-preprocessor", _write_json(tmp_path / "pp.json", cfg)])
    assert gf.read_gguf(str(tmp_path / "a.gguf")).image_proc == _expected(cfg, 64)
    args[1] = str(tmp_path / "b.gguf")
    cv.main(args)
    assert gf.read_gguf(str(tmp_path / "b.gguf")).image_proc is None
    with pytest.raises(ValueError, match="the model's img_size 64"):
        cv.main(args + ["--hf-preprocessor", _write_json(tmp_path / "pp224.json", tr.SiglipImageProcessorPil().to_dict())])


CLIP = {"do_resize": True, "size": {"shortest_edge": 224}, "resample": 3, "do_center_crop": True, "crop_size": {"height": 224, "width": 224},
        "do_rescale": True, "rescale_factor": 1 / 255, "do_normalize": True, "image_mean": [0.5] * 3, "image_std": [0.5] * 3}


@pytest.mark.parametrize("edit,field", [
    ({"do_resize": False}, "do_resize"),
    ({"size": {"longest_edge": 224}}, "longest_edge"),
    ({"size": {"shortest_edge": 224, "max_size": 300}}, "max_size"),
    ({"resample": 1}, "resample"),
    ({"resample": 0}, "resample"),
    ({"do_pad": True}, "do_pad"),
    ({"crop_size": {"height": 256, "width": 224}}, "crop_size"),
    ({"size": {"shortest_edge": 256}, "crop_size": {"height": 256, "width": 256}}, "img_size"),
    ({"do_center_crop": False}, "do_center_crop"),
    ({"size": {"height": 224, "width": 200}, "do_center_crop": False}, "img_size"),
])
def test_config_refusals_name_the_field(edit, field):
    with pytest.raises(ValueError, match=field):
        gf.image_proc_from_config(dict(CLIP, **edit), 224)


def test_config_mapping():
    """do_rescale / do_normalize false give 1.0 and (0, 1); integer sizes are a shortest edge and a square crop, as CLIP reads them."""
    d = gf.image_proc_from_config(dict(CLIP, do_rescale=False, do_normalize=False), 224)
    assert (d["rescale_factor"], d["mean"], d["std"]) == (1.0, [0.0] * 3, [1.0] * 3)
    d = gf.image_proc_from_config(dict(CLIP, size=224, crop_size=224), 224)
    assert (d["shortest_edge"], d["crop_height"], d["crop_width"]) == (224, 224, 224)
    assert gf.image_proc_from_config(d, 224) == d  # the struct's own fields pass through


GOOD = {"shortest_edge": 0, "height": 224, "width": 224, "crop_height": 0, "crop_width": 0, "resample": 3, "rescale_factor": 1 / 255,
        "mean": [0.5] * 3, "std": [0.5] * 3}


@pytest.mark.parametrize("edit,message", [
    ({"resample": 1}, "image_proc.resample = 1"),
    ({"resample": 0}, "image_proc.resample = 0"),
    ({"height": 0}, "image_proc.height / width = 0 x 224"),
    ({"shortest_edge": -1}, "image_proc.shortest_edge = -1"),
    ({"crop_height": 224}, "image_proc.crop_height / crop_width = 224 x 0"),
    ({"shortest_edge": 224}, "image_proc.shortest_edge = 224 without crop_height / crop_width"),
    ({"height": 200, "crop_height": 224, "crop_width": 224}, "image_proc.crop_height / crop_width = 224 x 224: larger than the resize target 200 x 224"),
    ({"height": 256, "width": 256}, "image_proc: the final size 256 x 256 (height x width) is not the model's img_size 224"),
    ({"shortest_edge": 256, "crop_height": 240, "crop_width": 240}, "image_proc: the final size 240 x 240 (crop_height x crop_width)"),
    ({"rescale_factor": 0.0}, "image_proc.rescale_factor = 0"),
    ({"rescale_factor": float("inf")}, "image_proc.rescale_factor = inf"),
    ({"mean": [0.5, float("nan"), 0.5]}, "image_proc.mean[1] = nan"),
    ({"std": [0.5, 0.5, 0.0]}, "image_proc.std[2] = 0"),
    ({"std": [float("inf"), 0.5, 0.5]}, "image_proc.std[0] = inf"),
])
def test_loader_refusals_name_the_field(edit, message, tmp_path):
    """A file's processor goes through vitb200_set_image_proc's checks before the device is touched: each refusal names the key."""
    vf = gf.read(_model_224(tmp_path))
    vf.image_proc = dict(GOOD, **edit)
    path = str(tmp_path / "bad.gguf")
    gf.write_gguf(path, vf)
    with pytest.raises(eng.VitB200Error) as ei:
        eng.vit_model_load(path, 0, 2)
    assert "vit." + message in str(ei.value), str(ei.value)


def test_loader_refuses_a_processor_for_a_vitstr_model(tmp_path):
    vf = gf.read(model_path("vitstr_micro", "f16"))
    vf.image_proc = dict(GOOD, height=96, width=96)
    path = str(tmp_path / "vitstr.gguf")
    gf.write_gguf(path, vf)
    with pytest.raises(eng.VitB200Error, match="vit.image_proc: this model takes 1-channel input"):
        eng.vit_model_load(path, 0, 2, head_tokens=25)


def test_loader_refuses_malformed_keys(tmp_path):
    """A mean of two values, or a processor key the loader does not know, fails the parse."""
    vf = gf.read(_model_224(tmp_path))
    vf.image_proc = dict(GOOD, mean=[0.5, 0.5])
    path = str(tmp_path / "short.gguf")
    with pytest.raises(ValueError):  # the writer packs exactly 3 floats
        gf.write_gguf(path, vf)
    vf.image_proc = GOOD
    gf.write_gguf(path, vf)
    raw = open(path, "rb").read()
    bad = raw.replace(b"vit.image_proc.image_std", b"vit.image_proc.image_sdd")
    (tmp_path / "sdd.gguf").write_bytes(bad)
    with pytest.raises(eng.VitB200Error, match="unknown key vit.image_proc.image_sdd"):
        eng.vit_model_load(str(tmp_path / "sdd.gguf"), 0, 2)
    # image_std as 3 float32 values re-labelled as int32: still 12 bytes, but not the array the key needs
    i = raw.index(b"vit.image_proc.image_std") + len(b"vit.image_proc.image_std")
    wrong = raw[:i + 4] + (5).to_bytes(4, "little") + raw[i + 8:]
    (tmp_path / "i32.gguf").write_bytes(wrong)
    with pytest.raises(eng.VitB200Error, match="vit.image_proc.image_std must be an array of 3 float32"):
        eng.vit_model_load(str(tmp_path / "i32.gguf"), 0, 2)


def test_gguf_parser_fuzzed_with_the_image_proc_keys(tmp_path):
    """tests/cpp/gguf_fuzz.cpp under ASan / UBSan with a file carrying every vit.image_proc.* key as its GGUF seed."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("no g++")
    exe = str(tmp_path / "gguf_fuzz")
    r = subprocess.run([gxx, "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-I", os.path.join(ROOT, "vit.cpp_b200", "csrc"), os.path.join(ROOT, "tests", "cpp", "gguf_fuzz.cpp"), "-o", exe],
                       capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr.lower():
        pytest.skip("sanitizer runtime not available: " + r.stderr[-200:])
    assert r.returncode == 0, r.stderr[-2000:]
    vf = gf.read(model_path("micro", "f16"))
    vf.image_proc = dict(GOOD, shortest_edge=72, height=0, width=0, crop_height=64, crop_width=64)
    seed = str(tmp_path / "seed.gguf")
    gf.write_gguf(seed, vf)
    assert b"vit.image_proc.image_mean" in open(seed, "rb").read()
    r = subprocess.run([exe, seed, model_path("micro", "f16")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert r.stdout.count("rejected") == 2


def test_kernels_build_for_sm90a_without_spills(tmp_path):
    """image_proc_h_kernel and image_proc_v_kernel alone, through nvcc -Xptxas -v for sm_90a: no spill stores or loads."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = tmp_path / "k.cu"
    src.write_text('#include "ptx.cuh"\n#include "preprocess.cuh"\n')
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", "-I",
                        os.path.join(ROOT, "vit.cpp_b200", "csrc"), str(src), "-o", str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    info = {}
    for m in re.finditer(r"Compiling entry function '\w*(image_proc_[hv]_kernel)\w*'.*?(\d+) bytes spill stores, (\d+) bytes spill loads",
                         r.stderr, re.S):
        info[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    assert info == {"image_proc_h_kernel": (0, 0), "image_proc_v_kernel": (0, 0)}, r.stderr
