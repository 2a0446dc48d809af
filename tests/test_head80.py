"""Models with 80-column attention heads (ViT-H/14 and the CLIP ViT-H/14 image towers) on the CPU: the CLIP converter accepts them
and the other converters still refuse them, the engine's load checks name each limit of head dim 80 before the device is touched, and
the emulation agrees with a float64 Hugging Face CLIPVisionModelWithProjection of that head dim."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.util import pkg, gf
from tests import clip_oracle as co
from tests import fp8_reference as fr
from tests.emulation_hd import Emulation
from tests.hf_oracle import init_model, save_and_convert

eng = pkg.engine
cv = pkg.convert

# name: (hidden, heads, layers, patch, image, projection dim); 2 heads of 80 columns
GEOMETRIES = {
    "h80_micro": (160, 2, 2, 16, 64, 96),     # 17 tokens: the split-precision form of the head-dim-80 attention
    "h80_h14": (160, 2, 2, 14, 224, 96),      # 257 tokens, ViT-H/14's at 224 px: its f16-operand form
}

# The emulation (f16 form, float64 accumulation) against the float64 HF oracle, max |a - b| / max |b| per image: the CLIP bound of
# tests/test_clip.py (measured 2-4e-4 at head dim 64).  Measured at head dim 80: 2.0-5.0e-4 (h80_micro image_embeds 5.0e-4, h80_h14
# 3.3e-4), the same f16 roundings of the GEMM operands and the soft-max table.
EMU_BOUND = 1e-3


def build_hf(geometry: str, seed: int = 0):
    """The float32 HF CLIP vision tower with projection (matrix weights f16-valued, QuickGELU) of a geometry of GEOMETRIES."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    D, H, L, P, S, proj = GEOMETRIES[geometry]
    cfg = CLIPVisionConfig(hidden_size=D, intermediate_size=4 * D, num_attention_heads=H, num_hidden_layers=L, patch_size=P, image_size=S,
                           projection_dim=proj, hidden_act="quick_gelu", layer_norm_eps=1e-5)
    return init_model(CLIPVisionModelWithProjection, cfg, seed, norms=("layer_norm", "layrnorm"), f32=("position_embedding",))


@pytest.fixture(scope="module", params=list(GEOMETRIES))
def clip80(request, tmp_path_factory):
    d = str(tmp_path_factory.mktemp(request.param))
    m = build_hf(request.param)
    path = save_and_convert(m, d, "clip")
    S = GEOMETRIES[request.param][4]
    imgs = gf.synthetic_images(3, S, seed=3)
    return request.param, m, d, path, gf.read_gguf(path), imgs, co.hf_outputs(m, imgs)


def test_clip_converter_takes_head_dim_80(clip80):
    geometry, m, d, path, vf, _, _ = clip80
    D, H, L, P, S, proj = GEOMETRIES[geometry]
    assert (vf.hidden_size, vf.num_attention_heads, vf.num_hidden_layers, vf.num_classes, vf.patch_size, vf.img_size) == (D, H, L, proj, P, S)
    assert vf.hidden_size // vf.num_attention_heads == 80
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    qkv = np.asarray(vf.tensors["blocks.1.attn.qkv.weight"], np.float32)
    for i, x in enumerate("qkv"):
        assert np.array_equal(qkv[i * D:(i + 1) * D], sd[f"vision_model.encoder.layers.1.self_attn.{x}_proj.weight"])


def test_clip_model_config_converts_through_the_cli(clip80, tmp_path):
    """A CLIPModel checkpoint: its config nests the vision tower's fields, and its text tower is ignored."""
    geometry, m, d, _, _, _, _ = clip80
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    full = dict(sd, **{"text_model.embeddings.token_embedding.weight": np.zeros((8, 4), np.float32), "logit_scale": np.zeros((), np.float32),
                       "text_projection.weight": np.zeros((4, 4), np.float32)})
    src = str(tmp_path / "model.safetensors")
    cv.write_safetensors(src, full)
    cfgp = co.write_config(str(tmp_path), vision_config={"hidden_act": "quick_gelu", "num_attention_heads": 2, "layer_norm_eps": 1e-5},
                           text_config={"hidden_act": "quick_gelu", "num_attention_heads": 1})
    out = str(tmp_path / "clip-h.gguf")
    cv.main([src, out, "--hf-config", cfgp])
    assert open(out, "rb").read() == open(os.path.join(d, "clip.gguf"), "rb").read()


@pytest.mark.parametrize("D,heads,hd", [(160, 5, 32), (144, 2, 72)])
def test_clip_converter_refuses_other_head_dims(D, heads, hd):
    sd = {"vision_model.embeddings.patch_embedding.weight": np.zeros((D, 3, 16, 16), np.float32)}
    with pytest.raises(ValueError, match=f"head dim {hd} is not supported"):
        cv.clip_to_timm(sd, {"num_attention_heads": heads})


def test_other_converters_still_refuse_head_dim_80():
    """DINOv2, SigLIP and the text towers: the engine has no head-dim-80 kernel for what they need (the map head's attention, the
    causal mask), so their converters refuse it as before."""
    pw = np.zeros((160, 3, 14, 14), np.float32)
    with pytest.raises(ValueError, match="head dim 80 is not supported"):
        cv.dinov2_to_timm({"embeddings.patch_embeddings.projection.weight": pw}, {"num_attention_heads": 2})
    with pytest.raises(ValueError, match="head dim 80 is not supported"):
        cv.siglip_to_timm({"vision_model.embeddings.patch_embedding.weight": pw}, {"num_attention_heads": 2})
    with pytest.raises(ValueError, match="head dim 80 is not supported"):
        cv.text_to_timm({"text_model.embeddings.token_embedding.weight": np.zeros((8, 160), np.float32)}, {"num_attention_heads": 2})


def _synthetic(tmp_path, hp):
    """A synthetic legacy-ggml model (hidden, layers, heads, patch, img), parsed."""
    path = str(tmp_path / "m.bin")
    gf.write_synthetic(path, hp, 1)
    return gf.read(path)


def _loads_or_lacks_a_device(vf):
    """Every shape check passes: the model loads on an H100, and fails only for the lack of a device elsewhere."""
    import torch
    if torch.cuda.is_available():
        eng.vit_model_from_tensors(vf, 0, 2).close()
        return
    with pytest.raises(eng.VitB200Error, match="no CUDA device"):
        eng.vit_model_from_tensors(vf, 0, 2)


@pytest.mark.parametrize("hp", [(160, 1, 2, 16, 64), (160, 1, 2, 14, 224), (160, 1, 2, 14, 336)])
def test_head_dim_80_models_pass_every_load_check(hp, tmp_path):
    """17, 257 and 577 tokens (ViT-H/14 at 224 and 336 px)."""
    _loads_or_lacks_a_device(_synthetic(tmp_path, hp))


def test_head_dim_80_token_limit(tmp_path):
    """640 tokens at head dim 80 (K and V of one head, 176-B rows, in 227 KB of shared memory): 626 tokens pass, 677 and DFN5B-H/14-378's
    730 are refused, naming the limit."""
    _loads_or_lacks_a_device(_synthetic(tmp_path, (160, 1, 2, 8, 200)))               # 25^2 + 1 = 626
    for hp, n in (((160, 1, 2, 8, 208), 677), ((160, 1, 2, 14, 378), 730)):
        with pytest.raises(eng.VitB200Error, match=f"{n} tokens not supported \\(max 640 at head dim 80"):
            eng.vit_model_from_tensors(_synthetic(tmp_path, hp), 0, 2)


def test_head_dim_80_refuses_the_map_head(tmp_path):
    """pool 2, the attention-pooling head: its attention kernel is 64 columns wide."""
    vf = _synthetic(tmp_path, (160, 1, 2, 16, 64))
    vf.pool = "map"   # patch rows only: no class token, no position row for it
    del vf.tensors["cls_token"]
    D = 160
    vf.tensors["pos_embed"] = np.ascontiguousarray(np.asarray(vf.tensors["pos_embed"]).reshape(-1, D)[1:][None])
    shapes = {"latent": (1, 1, D), "q.weight": (D, D), "q.bias": (D,), "kv.weight": (2 * D, D), "kv.bias": (2 * D,), "proj.weight": (D, D),
              "proj.bias": (D,), "norm.weight": (D,), "norm.bias": (D,), "mlp.fc1.weight": (4 * D, D), "mlp.fc1.bias": (4 * D,),
              "mlp.fc2.weight": (D, 4 * D), "mlp.fc2.bias": (D,)}
    for k, s in shapes.items():
        f16 = len(s) == 2
        vf.tensors["attn_pool." + k] = np.full(s, 0.01, np.float16 if f16 else np.float32)
        vf.tensor_ftype["attn_pool." + k] = int(f16)
    with pytest.raises(eng.VitB200Error, match="pool = 2 \\(map\\) not supported at head dim 80"):
        eng.vit_model_from_tensors(vf, 0, 2)


def test_other_head_dims_are_still_refused(tmp_path):
    for hp, hd in (((144, 1, 2, 16, 64), 72), ((128, 1, 4, 16, 64), 32), ((176, 1, 2, 16, 64), 88)):
        with pytest.raises(eng.VitB200Error, match=f"head dim {hd} not supported"):
            eng.vit_model_from_tensors(_synthetic(tmp_path, hp), 0, 2)


def test_head_dim_80_text_towers_are_refused():
    """The causal attention of the text towers is the 64-column wgmma kernel."""
    L = eng.lib()
    tok = np.zeros((8, 160), np.float16)
    ts = (eng.Tensor * 1)()
    ts[0].name, ts[0].data, ts[0].type, ts[0].n_dims = b"token_embd.weight", tok.ctypes.data, 1, 2
    ts[0].ne[0], ts[0].ne[1], ts[0].ne[2], ts[0].ne[3] = 160, 8, 1, 1
    hp = eng.Hparams(160, 1, 2, 96, 0, 0, 1, 1e-5)
    ta = eng.TextArch(16, 1, 1, 2, gf.ARCH_ACTIVATIONS.index("quick_gelu"), float("nan"), float("nan"))
    h = C.c_void_p()
    with pytest.raises(eng.VitB200Error, match="head dim 80 not supported"):
        eng._check(L.vitb200_create_text(C.byref(hp), C.byref(ta), ts, 1, 0, 2, 0, C.byref(h)), "vitb200_create_text")


@pytest.mark.parametrize("fp8", [False, True])
def test_emulation_at_head_dim_64_is_the_existing_one(fp8, tmp_path):
    """tests/emulation_hd.py only generalises the head split and the scale: at head dim 64 it gives tests/emulation.py's numbers."""
    from tests import emulation as base
    vf = _synthetic(tmp_path, (128, 2, 2, 16, 64))
    imgs = gf.synthetic_images(2, 64, seed=5)
    assert np.array_equal(Emulation(vf, fp8=fp8).forward(imgs), base.Emulation(vf, fp8=fp8).forward(imgs))


def test_emulation_matches_the_hf_oracle(clip80):
    """The emulation's head split and 1 / sqrtf(80) scale against float64 HF on embeds, pooler output and every hidden state."""
    geometry, _, _, _, vf, imgs, o = clip80
    emu = Emulation(vf, acc=np.float64, fp8=False)
    L = vf.num_hidden_layers
    x = {i: emu.encode(imgs, i) for i in range(L + 1)}
    d = {"image_embeds": fr.rel_dist(emu.forward(imgs), o["image_embeds"]).max(),
         "pooler_output": fr.rel_dist(emu.prelogits(x[L]), o["pooler_output"]).max()}
    d.update({f"hidden_states[{i}]": fr.rel_dist(x[i], o["hidden_states"][i]).max() for i in x})
    print(geometry, {k: f"{v:.2e}" for k, v in d.items()})
    assert max(d.values()) <= EMU_BOUND, d


def test_a_wrong_scale_fails_the_oracle_check(clip80):
    """The emulation with head dim 64's 1/8 in place of 1 / sqrt(80) is far outside the bound: the check sees the scale."""
    geometry, _, _, _, vf, imgs, o = clip80
    emu = Emulation(vf, acc=np.float64, fp8=False)
    for blk in emu.blocks:   # q scaled by sqrt(80) / 8 gives scores scaled by 1/8 in the emulation's 1 / sqrt(80) product
        D = vf.hidden_size
        k = np.float32(np.sqrt(80.0) / 8.0)
        blk["attn.qkv.bias"] = blk["attn.qkv.bias"].copy()
        blk["attn.qkv.bias"][:D] *= k
        w = blk["attn.qkv.weight"].copy()
        w[:D] *= k
        blk["attn.qkv.weight"] = w
    assert fr.rel_dist(emu.forward(imgs), o["image_embeds"]).max() > 10 * EMU_BOUND
