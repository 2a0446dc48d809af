"""SigLIP So400m-shaped towers without a GPU: the converter (head dim 72, F from the weights, the config's image_size over a floor grid),
the engine's load checks that refuse what head dim 72, F and the floor grid do not cover before the device is touched, and the emulation of
tests/so400m_oracle.py against float64 Hugging Face."""
import copy
import ctypes as C

import numpy as np
import pytest

from tests.util import pkg, gf
from tests import siglip_oracle as sgo
from tests import so400m_oracle as so
from tests import text_oracle as to
from tests import fp8_reference as fr
from tests.hf_oracle import save_and_convert

eng, cv = pkg.engine, pkg.convert

# float64 emulation vs float64 HF: the f16 roundings of the engine alone
EMU_BOUND = 1e-3

_built = {}


def _case(geo, classifier, tmp_path_factory):
    key = (geo, classifier)
    if key not in _built:
        d = str(tmp_path_factory.mktemp(f"{geo}_{classifier}"))
        m = so.build_hf(geo, classifier)
        path = save_and_convert(m, d, "siglip")
        vf = gf.read_gguf(path)
        imgs = gf.synthetic_images(2, vf.img_size, seed=3)
        _built[key] = (path, vf, imgs, sgo.hf_outputs(m, imgs))
    return _built[key]


@pytest.mark.parametrize("geo", list(so.GEOMETRIES))
def test_converter_round_trip(geo, tmp_path_factory):
    D, H, F, P, S = so.GEOMETRIES[geo]
    for classifier in (False, True):
        _, vf, _, _ = _case(geo, classifier, tmp_path_factory)
        G = S // P
        assert (vf.hidden_size, vf.num_attention_heads, vf.patch_size, vf.img_size) == (D, H, P, S)
        assert vf.pool == ("mean" if classifier else "map") and vf.n_tokens == G * G
        assert np.asarray(vf.tensors["pos_embed"]).reshape(-1, D).shape[0] == G * G
        for i in range(so.LAYERS):
            assert vf.tensors[f"blocks.{i}.mlp.fc1.weight"].shape == (F, D) and vf.tensors[f"blocks.{i}.mlp.fc2.weight"].shape == (D, F)
        if not classifier:
            assert vf.tensors["attn_pool.mlp.fc1.weight"].shape == (F, D)


def test_text_converter_round_trip(tmp_path):
    V, D, H, F, N, E = so.TEXT
    vf = gf.read_gguf(to.convert(so.build_text(), str(tmp_path)))
    assert (vf.hidden_size, vf.num_attention_heads, vf.num_classes) == (D, H, E)
    assert vf.text["causal"] == 0 and vf.text["pool"] == "last" and vf.text["context"] == N
    assert vf.tensors["blocks.1.mlp.fc1.weight"].shape == (F, D)


def test_converter_refuses_a_config_that_disagrees_with_the_weights():
    m = so.build_hf("micro72")
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    cfg = m.config.to_dict()
    with pytest.raises(ValueError, match="intermediate_size 4304 is not supported: the weights' mlp.fc1 has 576 rows"):
        cv.siglip_to_timm(sd, dict(cfg, intermediate_size=4304))
    with pytest.raises(ValueError, match="image_size 80: 16 position rows"):
        cv.siglip_to_timm(sd, dict(cfg, image_size=80))
    with pytest.raises(ValueError, match="head dim 48 is not supported"):
        cv.siglip_to_timm(sd, dict(cfg, num_attention_heads=3))


def _loads_or_lacks_a_device(vf):
    import torch
    if torch.cuda.is_available():
        eng.vit_model_from_tensors(vf, 0, 2).close()
        return
    with pytest.raises(eng.VitB200Error, match="no CUDA device"):
        eng.vit_model_from_tensors(vf, 0, 2)


@pytest.mark.parametrize("geo", list(so.GEOMETRIES))
def test_every_geometry_passes_the_load_checks(geo, tmp_path_factory):
    for classifier in (False, True):
        _loads_or_lacks_a_device(_case(geo, classifier, tmp_path_factory)[1])


def _with_width(vf, F, blocks=None, head=True):
    """vf with the MLP of `blocks` (default all) and, when `head`, of the pooling head F wide."""
    t = dict(vf.tensors)
    D = vf.hidden_size
    names = [f"blocks.{i}.mlp." for i in (range(vf.num_hidden_layers) if blocks is None else blocks)] + (["attn_pool.mlp."] if head else [])
    for p in names:
        t[p + "fc1.weight"] = np.full((F, D), 0.01, np.float16)
        t[p + "fc1.bias"] = np.zeros(F, np.float32)
        t[p + "fc2.weight"] = np.full((D, F), 0.01, np.float16)
    out = copy.copy(vf)
    out.tensors, out.tensor_ftype = t, dict(vf.tensor_ftype)
    return out


def test_mlp_width_refusals(tmp_path_factory):
    _, vf, _, _ = _case("micro72_p14", False, tmp_path_factory)
    _loads_or_lacks_a_device(_with_width(vf, 1152))                      # 8 D
    cases = [(_with_width(vf, 460), "pool = 2: F = 460 is not a multiple of 8"),
             (_with_width(vf, 1160), "pool = 2: F = 1160 out of range \\(8..1152 = 8 D\\)"),
             (_with_width(vf, 472, blocks=[1], head=False), "pool = 2: block 1's mlp.fc1 \\[472\\]\\[144\\]"),
             (_with_width(vf, 472, blocks=[], head=True), "'attn_pool.mlp.fc1.weight' \\[472\\]\\[144\\] disagrees with the blocks' F = 464")]
    for bad, msg in cases:
        with pytest.raises(eng.VitB200Error, match=msg):
            eng.vit_model_from_tensors(bad, 0, 2)


def test_token_limit_at_head_dim_72(tmp_path_factory):
    """800 tokens at head dim 72 (144-B rows): So400m at 448 px (1024 tokens) is refused, naming the limit; 800 itself is not above it."""
    _, vf, _, _ = _case("micro72", True, tmp_path_factory)
    for S, P, n in ((448, 14, 1024), (464, 16, 841)):
        big = _with_width(vf, 576, blocks=[], head=False)
        big.img_size, big.patch_size = S, P
        big.tensors["pos_embed"] = np.zeros((1, n, 144), np.float32)
        big.tensors["patch_embed.proj.weight"] = np.zeros((144, 3, P, P), np.float16)
        with pytest.raises(eng.VitB200Error, match=f"{n} tokens not supported \\(max 800 at head dim 72"):
            eng.vit_model_from_tensors(big, 0, 2)


def test_head_dim_72_and_the_floor_grid_are_for_siglip_pools_only(tmp_path):
    path = str(tmp_path / "m.bin")
    gf.write_synthetic(path, (144, 1, 2, 16, 64), 1)
    with pytest.raises(eng.VitB200Error, match="head dim 72 not supported \\(64 or 80; 72 with pools 2 map and 3 mean"):
        eng.vit_model_from_tensors(gf.read(path), 0, 2)
    gf.write_synthetic(path, (128, 1, 2, 14, 64), 1)
    vf = gf.read(path)
    vf.img_size = 64    # a 4 x 4 grid of 14-px patches would drop 8 pixels: pools 0 and 1 refuse it
    with pytest.raises(eng.VitB200Error, match="img_size 64 not a multiple of patch_size 14"):
        eng.vit_model_from_tensors(vf, 0, 2)


def test_head_dim_72_and_the_floor_grid_are_refused_at_pool_1(tmp_path):
    """DINOv2's class-plus-patch-mean pool (1) takes neither: its towers have 64- or 80-column heads and dividing patches."""
    path = str(tmp_path / "m.bin")
    for hp, msg in (((144, 1, 2, 16, 64), "head dim 72 not supported"), ((128, 1, 2, 14, 64), "img_size 64 not a multiple of patch_size 14")):
        gf.write_synthetic(path, hp, 1)
        vf = gf.read(path)
        vf.pool = "cls_patch_mean"
        vf.img_size = 64
        D = hp[0]
        vf.tensors["head.weight"] = np.full((vf.num_classes, 2 * D), 0.01, np.float16)
        with pytest.raises(eng.VitB200Error, match=msg):
            eng.vit_model_from_tensors(vf, 0, 2)


@pytest.mark.parametrize("classifier", [False, True])
def test_floor_grid_needs_img_size_multiple_of_4_at_vector_patch_sizes(classifier, tmp_path_factory):
    """Patch 16 reads pixel rows in 16-byte loads: a floor grid there needs img_size % 4 == 0.  micro72 (patch 16, a 4 x 4 grid) at 70 px
    is refused before the device is touched, naming the limit; at 68 px it loads; patch 14 (micro72_p14) takes any size."""
    _, vf, _, _ = _case("micro72", classifier, tmp_path_factory)
    bad = copy.copy(vf)
    bad.img_size = 70
    with pytest.raises(eng.VitB200Error, match="img_size 70 not supported with patch_size 16: a floor grid needs img_size % 4 == 0"):
        eng.vit_model_from_tensors(bad, 0, 2)
    ok = copy.copy(vf)
    ok.img_size = 68
    _loads_or_lacks_a_device(ok)
    _, vf14, _, _ = _case("micro72_p14", classifier, tmp_path_factory)
    odd = copy.copy(vf14)
    odd.img_size = 69
    _loads_or_lacks_a_device(odd)


def test_causal_text_towers_are_refused_at_head_dim_72():
    L = eng.lib()
    tok = np.zeros((8, 144), np.float16)
    ts = (eng.Tensor * 1)()
    ts[0].name, ts[0].data, ts[0].type, ts[0].n_dims = b"token_embd.weight", tok.ctypes.data, 1, 2
    ts[0].ne[0], ts[0].ne[1], ts[0].ne[2], ts[0].ne[3] = 144, 8, 1, 1
    hp = eng.Hparams(144, 1, 2, 96, 0, 0, 1, 1e-5)
    ta = eng.TextArch(16, 1, 1, 2, gf.ARCH_ACTIVATIONS.index("quick_gelu"), float("nan"), float("nan"))
    h = C.c_void_p()
    with pytest.raises(eng.VitB200Error, match="head dim 72 not supported \\(64; 72 with causal = 0"):
        eng._check(L.vitb200_create_text(C.byref(hp), C.byref(ta), ts, 1, 0, 2, 0, C.byref(h)), "vitb200_create_text")


@pytest.mark.parametrize("geo", ["micro72", "micro72_p14", "so400m_384"])
def test_emulation_matches_the_hf_oracle(geo, tmp_path_factory):
    """The emulation's 72-column heads, F and floor grid against float64 HF; taking the G P x G P window from the bottom-right corner
    (the dropped pixels in, the first ones out) is far outside the bound."""
    for classifier in (False, True):
        _, vf, imgs, o = _case(geo, classifier, tmp_path_factory)
        emu = so.Emulation(vf, acc=np.float64, fp8=False)
        L = vf.num_hidden_layers
        x = {i: emu.encode(imgs, i) for i in (0, L)}
        d = {"logits": fr.rel_dist(emu.forward(imgs), o["logits"]).max(), "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["prelogits"]).max()}
        d.update({f"hidden_states[{i}]": fr.rel_dist(x[i], o["hidden_states"][i]).max() for i in x})
        print(geo, classifier, {k: f"{v:.2e}" for k, v in d.items()})
        assert max(d.values()) <= EMU_BOUND, d
        cut = vf.img_size - vf.img_size // vf.patch_size * vf.patch_size
        if cut:
            wrong = so.Emulation(vf, crop=(cut, cut), acc=np.float64, fp8=False)
            assert fr.rel_dist(wrong.encode(imgs, 0), o["hidden_states"][0]).max() > 100 * EMU_BOUND
