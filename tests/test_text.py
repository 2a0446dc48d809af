"""CLIP and SigLIP text towers (vitb200_create_text) on the CPU: the converter's round trips for the five Hugging Face classes and its
refusals, the loader's refusals (which come before the device is touched), the GGUF parser fuzzed with the vit.text.* keys, the new
symbols, the new kernels compiled for sm_90a without spills, and the numpy emulation of the text schedule against float64 HF models."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests.util import pkg, gf
from tests import text_oracle as to
from tests.fp8_reference import rel_dist

eng = pkg.engine
cv = pkg.convert
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _clip_model(tmp_path, kind):
    """The five HF classes, tiny: (model, expected projection rows, has logit_scale, has logit_bias)."""
    import transformers as tr
    from tests.hf_oracle import init_model
    tc = to.clip_text_config("micro")
    if kind == "CLIPTextModel":
        return to.build_clip(projection=False), tc.hidden_size, False, False
    if kind == "CLIPTextModelWithProjection":
        return to.build_clip(), tc.projection_dim, False, False
    if kind == "SiglipTextModel":
        return to.build_siglip(), 128, False, False
    vision = dict(hidden_size=64, intermediate_size=256, num_hidden_layers=1, num_attention_heads=1, image_size=32, patch_size=16)
    if kind == "CLIPModel":
        cfg = tr.CLIPConfig(text_config=tc.to_dict(), vision_config=vision, projection_dim=96)
        return init_model(tr.CLIPModel, cfg, 0, norms=("layer_norm",), f32=("position_embedding",)), 96, True, False
    cfg = tr.SiglipConfig(text_config=to.siglip_text_config().to_dict(), vision_config=vision)
    return init_model(tr.SiglipModel, cfg, 0, norms=("layer_norm",), f32=("position_embedding",)), 128, True, True


@pytest.mark.parametrize("kind", ["CLIPTextModel", "CLIPTextModelWithProjection", "CLIPModel", "SiglipTextModel", "SiglipModel"])
def test_converter_round_trip(kind, tmp_path):
    m, E, scale, bias = _clip_model(tmp_path, kind)
    vf = gf.read_gguf(to.convert(m, str(tmp_path)))
    siglip = kind.startswith("Siglip")
    V, D, H, L, N, _ = to.GEOMETRIES["siglip64" if siglip else "micro"]
    assert (vf.hidden_size, vf.num_attention_heads, vf.num_hidden_layers, vf.num_classes, vf.patch_size, vf.img_size) == (D, H, L, E, 0, 0)
    assert len(vf.tensors) == 12 * L + 6
    assert vf.text["context"] == N and vf.text["causal"] == (0 if siglip else 1)
    assert vf.text["pool"] == ("last" if siglip else "eos_argmax")  # HF's default CLIP eos_token_id is 2
    assert vf.activation == ("gelu_pytorch_tanh" if siglip else "quick_gelu")
    assert (vf.text["logit_scale"] is not None, vf.text["logit_bias"] is not None) == (scale, bias)
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    if scale:
        assert vf.text["logit_scale"] == np.float32(sd["logit_scale"].reshape(-1)[0])
    assert np.array_equal(vf.tensors["token_embd.weight"], sd["text_model.embeddings.token_embedding.weight"].astype(np.float16))
    assert vf.tensors["pos_embed"].shape == (1, N, D)
    assert vf.tensors["head.weight"].shape == (E, D)
    if kind == "CLIPTextModel":
        assert np.array_equal(vf.tensors["head.weight"], np.eye(D, dtype=np.float16))
    if not siglip:
        assert not vf.tensors["head.bias"].any()


def test_converter_picks_eos_when_eos_token_id_is_not_2(tmp_path):
    vf = gf.read_gguf(to.convert(to.build_clip(eos_token_id=999), str(tmp_path)))
    assert (vf.text["pool"], vf.text["eos_token_id"]) == ("eos", 999)


@pytest.mark.parametrize("edit,message", [
    ({"num_attention_heads": 1}, "head dim 128"),
    ({"max_position_embeddings": 248}, "context 248"),
    ({"intermediate_size": 384}, "intermediate size 384"),
    ({"hidden_act": "relu"}, "hidden_act 'relu'"),
])
def test_converter_refusals_name_the_value(edit, message, tmp_path):
    import transformers as tr
    from tests.hf_oracle import init_model
    cfg = to.clip_text_config("micro").to_dict()
    cfg.update(edit)
    if edit.get("hidden_act") == "relu":  # HF builds the model; the converter refuses the config
        m = to.build_clip(projection=False)
        m.config.hidden_act = "relu"
    else:
        m = init_model(tr.CLIPTextModel, tr.CLIPTextConfig(**cfg), 0, norms=("layer_norm",), f32=("position_embedding",))
    with pytest.raises(ValueError, match=re.escape(message)):
        to.convert(m, str(tmp_path))


def _text_file(tmp_path, name="t.gguf", edit=None):
    vf = gf.read_gguf(to.convert(to.build_clip(), str(tmp_path / "src")))
    if edit:
        edit(vf)
    path = str(tmp_path / name)
    gf.write_gguf(path, vf)
    return path, vf


def _refused(path, match):
    with pytest.raises(eng.VitB200Error, match=match):
        eng.vit_model_load(path, 0, 2)


def test_loader_refusals(tmp_path):
    """Each refusal names the limit, before the device is touched."""
    path, vf = _text_file(tmp_path)
    raw = open(path, "rb").read()
    # an unknown vit.text.* key, and an unknown pool
    (tmp_path / "k.gguf").write_bytes(raw.replace(b"vit.text.eos_token_id", b"vit.text.eos_token_ix"))
    _refused(str(tmp_path / "k.gguf"), "unknown key vit.text.eos_token_ix")
    (tmp_path / "p.gguf").write_bytes(raw.replace(b"eos_argmax", b"eos_argmix"))
    _refused(str(tmp_path / "p.gguf"), "unknown vit.text.pool 'eos_argmix'")
    # an image key on a text file
    (tmp_path / "i.gguf").write_bytes(raw.replace(b"vit.text.causal", b"vit.layer_scale"))
    _refused(str(tmp_path / "i.gguf"), "must not carry the image key vit.layer_scale")
    # tensor counts
    p2, _ = _text_file(tmp_path, "n.gguf", lambda v: v.tensors.pop("blocks.1.norm1.bias"))
    _refused(p2, "model file has 29 tensors, but 30 tensors were expected")
    # context against pos_embed
    p3, _ = _text_file(tmp_path, "c.gguf", lambda v: v.text.update(context=15))
    _refused(p3, "vitb200_text_arch.context = 15, but 'pos_embed' has 16 rows")
    p4, _ = _text_file(tmp_path, "c2.gguf", lambda v: v.text.update(context=225))
    _refused(p4, r"vitb200_text_arch.context = 225 out of range \(1..224")
    # SwiGLU
    p5, _ = _text_file(tmp_path, "a.gguf", lambda v: setattr(v, "activation", "swiglu"))
    _refused(p5, "vitb200_text_arch.activation = 4 out of range")
    # head_tokens
    with pytest.raises(eng.VitB200Error, match="head_tokens must be 1"):
        eng.vit_model_load(path, 0, 2, head_tokens=2)


def test_create_text_refusals(tmp_path):
    """vitb200_create_text with a caller-built list: patch_size / img_size, the token table's shape, V >= 1."""
    _, vf = _text_file(tmp_path)
    vf.patch_size = 16
    with pytest.raises(eng.VitB200Error, match="patch_size and img_size must be 0"):
        eng.vit_model_from_tensors(vf)
    vf.patch_size = 0
    with pytest.raises(eng.VitB200Error, match=r"'token_embd.weight' must be \[V\]\[128\]"):
        eng.vit_model_from_tensors(vf, edit=lambda es: [e if e[0] != "token_embd.weight" else [e[0], e[1][:, :64].copy(), e[2], [64, e[1].shape[0]]]
                                                        for e in es])
    with pytest.raises(eng.VitB200Error, match="missing tensor 'token_embd.weight'"):
        eng.vit_model_from_tensors(vf, edit=lambda es: [e for e in es if e[0] != "token_embd.weight"])


def test_writer_refuses_image_fields_on_a_text_file(tmp_path):
    _, vf = _text_file(tmp_path)
    vf.pre_norm = 1
    with pytest.raises(ValueError, match="a text tower has no pre-norm"):
        gf.write_gguf(str(tmp_path / "x.gguf"), vf)


def test_gguf_parser_fuzzed_with_the_text_keys(tmp_path):
    """tests/cpp/gguf_fuzz.cpp under ASan / UBSan with a text file as its GGUF seed."""
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
    seed, _ = _text_file(tmp_path, edit=lambda v: v.text.update(logit_scale=2.5, logit_bias=-10.0))
    assert b"vit.text.logit_bias" in open(seed, "rb").read()
    r = subprocess.run([exe, seed], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert r.stdout.count("rejected") == 1


def test_text_symbols_are_exported():
    names = {"vitb200_create_text", "vitb200_get_text_arch", "vitb200_encode_text", "vitb200_encode_text_device",
             "vitb200_test_attention_hilo_causal"}
    assert names <= set(eng.declared_symbols())
    L = eng.lib()
    assert all(hasattr(L, n) for n in names)


def test_kernels_build_for_sm90a_without_spills(tmp_path):
    """The causal attention, the token gather and the text pool kernels through nvcc -Xptxas -v for sm_90a: no spills."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = tmp_path / "k.cu"
    src.write_text('#include "attention_wgmma.cuh"\n'
                   "template __global__ void vitb200::attention_wgmma_kernel<true>(const __grid_constant__ CUtensorMap, const __grid_constant__ "
                   "CUtensorMap, const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap, __half *, int, int, int, int, float);\n"
                   "template __global__ void vitb200::text_pool_kernel<4>(const float *, const int32_t *, int, int, int, int, const float *, "
                   "const float *, __half *, int, float);\n"
                   "template __global__ void vitb200::text_pool_kernel<8>(const float *, const int32_t *, int, int, int, int, const float *, "
                   "const float *, __half *, int, float);\n"
                   "template __global__ void vitb200::text_pool_kernel<16>(const float *, const int32_t *, int, int, int, int, const float *, "
                   "const float *, __half *, int, float);\n")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", "-I",
                        os.path.join(ROOT, "vit.cpp_b200", "csrc"), str(src), "-o", str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    info = {}
    for m in re.finditer(r"Compiling entry function '(\w*(?:attention_wgmma_kernelILb1|text_pool_kernelILi\d+|token_embed_kernel)\w*)'.*?"
                         r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr, re.S):
        info[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    assert len(info) == 5, r.stderr
    assert set(info.values()) == {(0, 0)}, info


def _emulation_distances(model, vf, ids, projection=True):
    hf = to.hf_outputs(model, ids)
    em = to.TextEmulation(vf, fp8=False)
    x = [em.encode_ids(ids, layers=i) for i in range(vf.num_hidden_layers + 1)]
    d = {"embeds": rel_dist(em.embeds(ids), hf["embeds"]).max()}
    if projection:
        d["pooled"] = rel_dist(em.pooled(ids, x[-1]), hf["pooled"]).max()
    for i, h in enumerate(hf["hidden_states"]):
        d[f"hidden_states[{i}]"] = rel_dist(x[i], h).max()
    d["last_hidden_state"] = rel_dist(em.final_ln(x[-1]), hf["last_hidden_state"]).max()
    return d


# (model, eos_token_id of the config, id that ends each sequence): CLIP's two EOS modes and SigLIP's last row
EMULATION_CASES = [("clip_quick_gelu_argmax", 2), ("clip_gelu_eos", 999), ("clip_ctx77_argmax", 2), ("siglip", None)]


def build_case(name):
    """(HF model, sequence-end id, eos_at list) of an EMULATION_CASES entry; the end id is the largest id for eos_argmax."""
    if name == "siglip":
        return to.build_siglip(), None
    if name == "clip_gelu_eos":
        return to.build_clip(activation="gelu_erf", eos_token_id=999), 999
    return to.build_clip("ctx77" if "77" in name else "micro"), to.GEOMETRIES["ctx77" if "77" in name else "micro"][0] - 1


@pytest.mark.parametrize("name,_eos", EMULATION_CASES)
def test_emulation_against_hugging_face(name, _eos, tmp_path):
    """The emulation of the text schedule against float64 HF: every distance is the f16 noise floor of the emulation's roundings (a
    wrong mask, pool or gather is orders of magnitude away).  EOS first, last, absent; padding ids vary after it."""
    model, end = build_case(name)
    vf = gf.read_gguf(to.convert(model, str(tmp_path)))
    N, V = vf.text["context"], to.GEOMETRIES["ctx77" if "77" in name else ("siglip64" if name == "siglip" else "micro")][0]
    rng = np.random.default_rng(5)
    ids = to.padded_ids(rng, 4, N, V, end if end is not None else V - 1, [0, N - 1, 5, None])
    if end is not None and end == V - 1:
        ids[3, 9] = end  # a second maximum after the first in row 2 ...
        ids[2, 9] = end  # ... the first occurrence (position 5) wins
        ids[3, :] = np.minimum(ids[3], V - 2)  # row 3: no end id, argmax of the random ids
    d = _emulation_distances(model, vf, ids, projection=True)
    print(name, {k: f"{v:.2e}" for k, v in d.items()})
    assert max(d.values()) < 2e-2, d
