"""Models with 80-column attention heads on the GPU: the head-dim-80 attention kernel alone against float64, the forward pass against the
unmodified reference (tests/golden/h80_*.npz), the block-0 taps against the restatement, CLIP H-shaped towers against float64 Hugging
Face, non-finite isolation, and every image entry point."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np
import pytest

from oracle import restatement as rs
from tests import clip_oracle as co
from tests import fp8_reference as fr
from tests.emulation_hd import Emulation
from tests.hf_oracle import save_and_convert
from tests.test_gpu_forward import check_parity
from tests.test_gpu_fp8 import E2E_TOL
from tests.test_gpu_kernels import _attention_ref
from tests.test_head80 import GEOMETRIES, build_hf
from tests.util import pkg, gf

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_head80 as mg  # noqa: E402

eng = pkg.engine
pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HD = 80
MAX_TOKENS = 640   # the engine's limit at head dim 80 (ATT80_MAX_TOKENS)


HOOK_CASES = [(2, n, 2) for n in (1, 17, 64, 224, 225, 257, 577, MAX_TOKENS)] + [(24, 257, 16)]   # (B, N, H)


@pytest.mark.parametrize("split", [True, False], ids=["split", "f16"])
@pytest.mark.parametrize("B,N,H", HOOK_CASES)
def test_hook_against_numpy(B, N, H, split):
    """The head-dim-80 kernel alone, on random q | k | v with scores spread over several units: within the bound of the 64-column hook
    tests (2^-10 relative + 2e-3 of the largest output).  Split operands (N <= 224, as the engine runs them) against the restatement on
    the hi + lo values, f16 operands against it on the f16 values; (24, 257, 16) is ViT-H/14's problem count per image times 24."""
    if split and N > 224:
        with pytest.raises(eng.VitB200Error, match="needs N <= 224"):
            eng.test_attention_hd(np.zeros((B * N, 3 * H * HD), np.float32), B, N, H, HD, True)
        return
    rng = np.random.default_rng(N * 131 + H)
    qkv = rng.normal(0.0, 1.0, (B * N, 3 * H * HD)).astype(np.float32)
    qkv[:, : H * HD] *= 1.5
    out = eng.test_attention_hd(qkv, B, N, H, HD, split)
    if split:
        hi, lo = eng.split_hi_lo(qkv)
        seen = hi.astype(np.float32) + lo.astype(np.float32)
    else:
        seen = qkv.astype(np.float16).astype(np.float32)
    ref = _attention_ref(seen, B, N, H, HD)
    assert np.isfinite(out).all()
    err = np.abs(out - ref)
    tol = 2.0 ** -10 * np.abs(ref) + 2e-3 * np.abs(ref).max()
    assert (err <= tol).all(), (err.max(), np.abs(ref).max(), np.unravel_index(err.argmax(), err.shape))
    if split and N > 1:   # closer to the split-operand restatement than to the f16-operand one (one key: O = f16(v) either way)
        ref16 = _attention_ref(qkv.astype(np.float16), B, N, H, HD)
        assert np.abs(out - ref).mean() < 0.6 * np.abs(out - ref16).mean()


def test_hook_limits():
    with pytest.raises(eng.VitB200Error, match=f"{MAX_TOKENS + 1} tokens not supported \\(max {MAX_TOKENS} at head dim 80"):
        eng.test_attention_hd(np.zeros((MAX_TOKENS + 1, 3 * HD), np.float32), 1, MAX_TOKENS + 1, 1, HD, False)
    with pytest.raises(eng.VitB200Error, match="head dim 72 not supported"):
        eng.test_attention_hd(np.zeros((4, 3 * 72), np.float32), 1, 4, 1, 72, False)
    with pytest.raises(eng.VitB200Error, match="does not run head dim 80"):
        eng.test_attention_hd(np.zeros((4, 3 * HD), np.float32), 1, 4, 1, HD, False, eng.ATTN_MMA8)


def test_hook_at_head_dim_64_is_the_existing_kernels():
    rng = np.random.default_rng(5)
    qkv = rng.normal(0.0, 1.0, (2 * 197, 3 * 3 * 64)).astype(np.float32)
    assert np.array_equal(eng.test_attention_hd(qkv, 2, 197, 3, 64, False, eng.ATTN_MMA8),
                          eng.test_attention(qkv.astype(np.float16), 2, 197, 3, eng.ATTN_MMA8))
    assert np.array_equal(eng.test_attention_hd(qkv, 2, 197, 3, 64, True), eng.test_attention_hilo(qkv, 2, 197, 3))


_models = {}


def _model_path(name, tmp_path_factory):
    """The fixture's synthetic model file, checked against the sha256 the fixture was generated from."""
    if name not in _models:
        path = str(tmp_path_factory.mktemp(name) / f"{name}.bin")
        mg.write_model(path, name)
        g = np.load(os.path.join(GOLD, f"{name}_f16.npz"))
        assert hashlib.sha256(open(path, "rb").read()).hexdigest() == str(g["model_sha256"])
        _models[name] = path
    return _models[name]


@pytest.mark.parametrize("name", list(mg.CASES))
def test_logits_and_topk_match_the_reference(name, tmp_path_factory):
    """17 tokens (split-precision attention) and 257 (f16 operands), 8 images each, against the unmodified reference."""
    g = np.load(os.path.join(GOLD, f"{name}_f16.npz"))
    m = eng.vit_model_load(_model_path(name, tmp_path_factory), 0, 8)
    imgs = gf.synthetic_images(int(g["n_images"]), m.img_size, seed=int(g["image_seed"]))
    probs, idx, val, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    m.close()
    re = check_parity(logits, probs, idx, g["logits"], g["probs"])
    print(name, "max-norm error per image", np.array2string(re, precision=6))
    assert np.array_equal(idx, np.argsort(-g["logits"], 1, kind="stable")[:, :5])


@pytest.mark.parametrize("name", list(mg.CASES))
def test_block0_taps_match_the_restatement(name, tmp_path_factory):
    path = _model_path(name, tmp_path_factory)
    vf = gf.read(path)
    om = rs.OracleModel(vf, gf.tensor_specs)
    imgs = gf.synthetic_images(2, vf.img_size, seed=7)
    m = eng.vit_model_load(path, 0, 4)
    _, _, taps = eng.vit_predict_debug(m, imgs, 0)
    m.close()
    for b in range(2):
        _, _, t_o = om.forward(imgs[b], 0, tuple(eng.TAP_SHAPES))
        for tap, tol in [("embed", 1e-5), ("ln1", 2e-3), ("qkv", 2e-3), ("attn", 2e-3), ("x1", 2e-3), ("ln2", 2e-3),
                         ("h", 3e-3), ("x2", 2e-3), ("final_ln", 3e-3), ("x_final", 2e-3)]:
            a, r = taps[tap][b], t_o[tap]
            assert np.abs(a - r).max() <= tol * np.abs(r).max(), (tap, np.abs(a - r).max(), np.abs(r).max())


_clip = {}


def _clip_case(geometry, tmp_path_factory):
    if geometry not in _clip:
        d = str(tmp_path_factory.mktemp(geometry))
        m = build_hf(geometry)
        path = save_and_convert(m, d, "clip")
        vf = gf.read_gguf(path)
        imgs = gf.synthetic_images(3, vf.img_size, seed=3)
        o = co.hf_outputs(m, imgs)
        emu = Emulation(vf, acc=np.float64, fp8=False)
        L = vf.num_hidden_layers
        x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
        emu_d = {"logits": fr.rel_dist(emu.forward(imgs), o["image_embeds"]), "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["pooler_output"])}
        emu_d.update({f"tokens{i}": fr.rel_dist(x[i], o["hidden_states"][i]) for i in x})
        _clip[geometry] = (path, vf, imgs, o, emu_d)
    return _clip[geometry]


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_clip_tower_against_the_hf_oracle(geometry, tmp_path_factory):
    """image_embeds, pooler_output and hidden states 0, L-1, L within twice the emulation's distance of float64 HF."""
    path, vf, imgs, o, emu_d = _clip_case(geometry, tmp_path_factory)
    L, n = vf.num_hidden_layers, imgs.shape[0]
    m = eng.vit_model_load(path, 0, n)
    logits = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    assert m.last_launch_count() == 3 + 7 * L + 4
    got = {"logits": fr.rel_dist(logits, o["image_embeds"])}
    _, pre = eng.vit_features(m, imgs, layers=L, norm=True, tokens=False, prelogits=True)
    got["prelogits"] = fr.rel_dist(pre.reshape(n, -1), o["pooler_output"])
    for i in (0, L - 1, L):
        got[f"tokens{i}"] = fr.rel_dist(eng.vit_features(m, imgs, layers=i, norm=False)[0], o["hidden_states"][i])
    m.close()
    print(geometry, {k: f"{got[k].max():.2e} (emulation {emu_d[k].max():.2e})" for k in got})
    bad = {k: (got[k].max(), emu_d[k].max()) for k in got if got[k].max() > 2 * emu_d[k].max()}
    assert not bad, bad


def test_attention_profile_kind_counts_the_new_kernel(tmp_path_factory):
    """Profiling kind 6 (attention) times one launch per block with 4 N^2 D FLOPs per image."""
    path, vf, imgs, _, _ = _clip_case("h80_h14", tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3)
    L = eng.lib()
    eng._check(L.vitb200_profile_enable(m.handle, 1), "profile_enable")
    eng.vit_predict(m, imgs, 5)
    ms, cnt, fl = C.c_double(), C.c_int(), C.c_double()
    eng._check(L.vitb200_profile_read(m.handle, 6, C.byref(ms), C.byref(cnt), C.byref(fl)), "profile_read")
    eng._check(L.vitb200_profile_enable(m.handle, 0), "profile_enable")
    m.close()
    N, D = vf.n_tokens, vf.hidden_size
    assert cnt.value == vf.num_hidden_layers and ms.value > 0
    assert fl.value == 4.0 * 3 * N * N * D


@pytest.mark.parametrize("name", list(mg.CASES))
def test_a_nan_image_leaves_its_batch_mates_untouched(name, tmp_path_factory):
    """Image 2 of 5 holds a NaN pixel: the other four rows are bit-identical to a clean batch, on the eager call, the call that captures
    the graph and a replay."""
    m = eng.vit_model_load(_model_path(name, tmp_path_factory), 0, 5)
    imgs = gf.synthetic_images(5, m.img_size, seed=21)
    clean = eng.vit_predict(m, imgs, 5, want_logits=True)
    bad = imgs.copy()
    bad[2, -1, -1, -1] = np.nan
    rows = [0, 1, 3, 4]
    for call in range(3):
        out = eng.vit_predict(m, bad, 5, want_logits=True)
        for a, b in zip(out, clean):
            assert np.array_equal(a[rows], b[rows]), (name, call)
        assert not np.isfinite(out[3][2]).all()
    again = eng.vit_predict(m, imgs, 5, want_logits=True)
    m.close()
    for a, b in zip(again, clean):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_every_entry_point(geometry, tmp_path_factory):
    """From tensors == from the file; sharded and device forward == vit_predict; the u8 path == the f32 path on the images it returns,
    with and without an image processor; the FP8 engine within its end-to-end bound of the FP8 emulation."""
    import torch
    path, vf, imgs, _, _ = _clip_case(geometry, tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3)
    ref = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    mt = eng.vit_model_from_tensors(vf, 0, 3)
    assert np.array_equal(eng.vit_predict(mt, imgs, 5, want_logits=True)[3], ref)
    mt.close()
    assert np.array_equal(eng.vit_predict_sharded([m], imgs, 5)[0], eng.vit_predict(m, imgs, 5)[0])
    d_img = torch.from_numpy(imgs).cuda()
    d_log = torch.empty((3, vf.num_classes), dtype=torch.float32, device="cuda")
    eng._check(eng.lib().vitb200_forward_device(m.handle, d_img.data_ptr(), 3, None, d_log.data_ptr(), None, None, 0, None),
               "vitb200_forward_device")
    eng._check(eng.lib().vitb200_sync(m.handle), "vitb200_sync")
    assert np.array_equal(d_log.cpu().numpy(), ref)
    rng = np.random.default_rng(3)
    u8 = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((97, 131), (64, 64), (250, 233))]
    S = vf.img_size
    for proc in (None, {"do_resize": True, "size": {"shortest_edge": S}, "resample": 3, "do_center_crop": True,
                        "crop_size": {"height": S, "width": S}, "do_rescale": True, "rescale_factor": 1 / 255, "do_normalize": True,
                        "image_mean": [0.48145466, 0.4578275, 0.40821073], "image_std": [0.26862954, 0.26130258, 0.27577711]}):
        if proc is not None:
            m.set_image_proc(proc)
        f32, _, _, _, logits = eng.vit_image_preprocess_predict(m, u8)
        assert np.array_equal(logits, eng.vit_predict(m, f32, 5, want_logits=True)[3])
        tok = eng.vit_features_u8(m, u8, layers=1, norm=False)[0]
        assert np.array_equal(tok, eng.vit_features(m, f32, layers=1, norm=False)[0])
    m.close()
    m8 = eng.vit_model_load(path, 0, 3, fp8=True)
    logits8 = eng.vit_predict(m8, imgs, 5, want_logits=True)[3]
    m8.close()
    d = fr.rel_dist(logits8, Emulation(vf).forward(imgs))
    print(f"{geometry} FP8: GPU vs emulation {np.array2string(d, precision=4)} (bound {E2E_TOL:.4f})")
    assert d.max() <= E2E_TOL, d
