"""CLIP and SigLIP text towers on the GPU (vitb200_create_text): the causal wgmma attention against numpy, the engine against the float64
Hugging Face oracle within twice the emulation's own distance (tests/text_oracle.py), one call against two, the launch count, sequence
independence and the out-of-range id contract, the FP8 engine against its emulation, zero-shot logits against HF's logits_per_image, and
the refusals between image and text engines."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.util import pkg, gf
from tests import text_oracle as to
from tests.fp8_reference import rel_dist
from tests.test_gpu_fp8 import E2E_TOL

eng = pkg.engine
pytestmark = pytest.mark.gpu


def _attention64(qkv, B, N, H, causal):
    q, k, v = np.asarray(qkv, np.float64).reshape(B, N, 3, H, 64).transpose(2, 0, 3, 1, 4)
    s = np.einsum("bhqd,bhkd->bhqk", q, k) / 8.0
    if causal:
        s = np.where(np.tril(np.ones((N, N), bool)), s, -np.inf)
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    return np.einsum("bhqk,bhkd->bhqd", p, v).transpose(0, 2, 1, 3).reshape(B * N, H * 64)


@pytest.mark.parametrize("N", [1, 63, 64, 65, 77, 128, 224])
def test_causal_attention_hook(N):
    """The causal kernel against float64 (the f16 soft-max table and the f16 output are the noise), and the non-causal kernel's results
    unchanged against the same reference without the mask.  Row 0 attends to key 0 alone: its output is v_0 as the kernel holds it, hi + lo,
    rounded to f16."""
    B, H = 2, 2
    rng = np.random.default_rng(N)
    qkv = rng.standard_normal((B * N, 3 * H * 64)).astype(np.float32)
    out = eng.test_attention_hilo_causal(qkv, B, N, H)
    ref = _attention64(qkv, B, N, H, True)
    assert np.isfinite(out).all()
    assert np.abs(out - ref).max() <= 4e-3 * np.abs(ref).max() + 1e-3, np.abs(out - ref).max()
    v0 = qkv.reshape(B, N, 3, H * 64)[:, 0, 2]
    hi, lo = eng.split_hi_lo(v0)
    assert np.array_equal(out.reshape(B, N, -1)[:, 0], (hi.astype(np.float32) + lo.astype(np.float32)).astype(np.float16).astype(np.float32))
    full = eng.test_attention_hilo(qkv, B, N, H)
    assert np.abs(full - _attention64(qkv, B, N, H, False)).max() <= 4e-3 * np.abs(ref).max() + 1e-3
    if N > 1:
        assert not np.array_equal(full, out)


@pytest.fixture(scope="module")
def towers(tmp_path_factory):
    """(name -> (HF model, GGUF path, end id)) for CLIP in both EOS modes and SigLIP."""
    d = tmp_path_factory.mktemp("text")
    out = {}
    for name in ("clip_quick_gelu_argmax", "clip_gelu_eos", "clip_ctx77_argmax", "siglip"):
        from tests.test_text import build_case
        model, end = build_case(name)
        out[name] = (model, to.convert(model, str(d / name)), end)
    return out


def _ids(name, vf, B=6, seed=3):
    V = int(vf.tensors["token_embd.weight"].shape[0])
    N = vf.text["context"]
    end = V - 1 if vf.text["pool"] != "eos" else vf.text["eos_token_id"]
    rng = np.random.default_rng(seed)
    ids = to.padded_ids(rng, B, N, V, end, [0, N - 1, 4, None, 7, N // 2][:B])
    return ids


@pytest.mark.parametrize("name", ["clip_quick_gelu_argmax", "clip_gelu_eos", "clip_ctx77_argmax", "siglip"])
def test_against_hugging_face(towers, name):
    """embeds, the pooled rows (the final LayerNorm of every token row at the pooled positions) and hidden_states at every depth, each
    within twice the emulation's distance from float64 HF (and a 1e-4 floor)."""
    model, path, _ = towers[name]
    vf = gf.read_gguf(path)
    ids = _ids(name, vf)
    hf = to.hf_outputs(model, ids)
    em = to.TextEmulation(vf)
    m = eng.vit_model_load(path, 0, 8)
    assert m.text_arch["pool"] == vf.text["pool"] and m.text_arch["causal"] == vf.text["causal"]
    emb, tok = eng.vit_encode_text(m, ids, norm=True, tokens=True)
    x = [em.encode_ids(ids, i) for i in range(vf.num_hidden_layers + 1)]
    tol = lambda a, b: 2 * rel_dist(a, b).max() + 1e-4
    assert rel_dist(emb, hf["embeds"]).max() <= tol(em.embeds(ids), hf["embeds"])
    rows = to.pool_rows(ids, vf.text["pool"], vf.text["eos_token_id"])
    pooled = tok[np.arange(len(ids)), rows]
    assert rel_dist(pooled, hf["pooled"]).max() <= tol(em.pooled(ids, x[-1]), hf["pooled"])
    assert rel_dist(tok, hf["last_hidden_state"]).max() <= tol(em.final_ln(x[-1]), hf["last_hidden_state"])
    for i in range(vf.num_hidden_layers + 1):
        _, h = eng.vit_encode_text(m, ids, layers=i, norm=False, tokens=True, embeds=False)
        assert rel_dist(h, hf["hidden_states"][i]).max() <= tol(x[i], hf["hidden_states"][i]), i
    m.close()


def test_one_call_equals_two_and_launch_count(towers):
    """SDXL's case: hidden_states[-2] and embeds in one call equal two separate calls, bit for bit; embeds alone launch 1 + 7 L + 2."""
    _, path, _ = towers["clip_ctx77_argmax"]
    vf = gf.read_gguf(path)
    ids = _ids("clip_ctx77_argmax", vf)
    m = eng.vit_model_load(path, 0, 8)
    L = vf.num_hidden_layers
    emb, tok = eng.vit_encode_text(m, ids, layers=L - 1, norm=False, tokens=True)
    emb2, _ = eng.vit_encode_text(m, ids)
    assert m.last_launch_count() == 1 + 7 * L + 2
    _, tok2 = eng.vit_encode_text(m, ids, layers=L - 1, norm=False, tokens=True, embeds=False)
    assert np.array_equal(emb, emb2) and np.array_equal(tok, tok2)
    _, tok16 = eng.vit_encode_text(m, ids, layers=L - 1, norm=True, tokens=True, embeds=False, dtype=np.float16)
    assert m.last_launch_count() == 1 + 7 * (L - 1) + 1
    m.close()


@pytest.mark.parametrize("name", ["clip_gelu_eos", "siglip"])
def test_sequence_independence(towers, name):
    """Each sequence alone (eager, then graph-replayed on the next calls) equals its row in a mixed batch, bit for bit."""
    _, path, _ = towers[name]
    vf = gf.read_gguf(path)
    ids = _ids(name, vf)
    m = eng.vit_model_load(path, 0, 8)
    emb, tok = eng.vit_encode_text(m, ids, tokens=True, norm=False)
    for b in range(len(ids)):
        for _ in range(3):  # eager, capture, replay
            e1, t1 = eng.vit_encode_text(m, ids[b:b + 1], tokens=True, norm=False)
            assert np.array_equal(e1[0], emb[b]) and np.array_equal(t1[0], tok[b]), b
    m.close()


def test_out_of_range_ids(towers):
    """The device call gives NaN rows for a sequence holding id V, and only for it; the host call refuses the id, naming where it is."""
    _, path, _ = towers["clip_quick_gelu_argmax"]
    vf = gf.read_gguf(path)
    V = int(vf.tensors["token_embd.weight"].shape[0])
    ids = _ids("clip_quick_gelu_argmax", vf, B=4)
    m = eng.vit_model_load(path, 0, 8)
    ref, _ = eng.vit_encode_text(m, ids)
    bad = ids.copy()
    bad[2, 9] = V
    with pytest.raises(eng.VitB200Error, match=f"sequence 2, position 9: id {V} out of range"):
        eng.vit_encode_text(m, bad)
    d_ids = torch.from_numpy(bad).cuda()
    d_emb = torch.empty((4, m.embed_dim), dtype=torch.float32, device="cuda")
    d_tok = torch.empty((4, m.n_tokens, m.hidden_size), dtype=torch.float32, device="cuda")
    req = eng.FeaturesReq(vf.num_hidden_layers, 0, 0)
    eng._check(eng.lib().vitb200_encode_text_device(m.handle, d_ids.data_ptr(), 4, d_emb.data_ptr(), C.byref(req), d_tok.data_ptr(),
                                                   torch.cuda.current_stream().cuda_stream),
               "vitb200_encode_text_device")
    torch.cuda.synchronize()
    emb, tok = d_emb.cpu().numpy(), d_tok.cpu().numpy()
    assert np.isnan(emb[2]).all() and np.isnan(tok[2]).all()
    keep = [0, 1, 3]
    assert np.array_equal(emb[keep], ref[keep]) and np.isfinite(tok[keep]).all()
    m.close()


def test_fp8_against_its_emulation(towers):
    model, path, _ = towers["clip_ctx77_argmax"]
    vf = gf.read_gguf(path)
    ids = _ids("clip_ctx77_argmax", vf)
    m = eng.vit_model_load(path, 0, 8, fp8=True)
    emb, _ = eng.vit_encode_text(m, ids)
    em = to.TextEmulation(vf, fp8=True)
    ref = em.embeds(ids)
    d = rel_dist(emb, ref).max()
    print("fp8 text embeds vs emulation", d, "vs f16 HF", rel_dist(emb, to.hf_outputs(model, ids)["embeds"]).max())
    assert d <= E2E_TOL, d  # the image towers' FP8 bound: Hopper's e4m3 MMA adds with fewer than f32's mantissa bits
    m.close()


@pytest.mark.parametrize("family", ["clip", "siglip"])
def test_zero_shot(family, tmp_path):
    """A tiny CLIPModel / SiglipModel: both towers converted, images through the image engine and ids through the text engine;
    zero_shot_logits against HF's logits_per_image, with the same arg-max per image."""
    import transformers as tr
    from tests.hf_oracle import init_model
    vision = dict(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, image_size=64, patch_size=16,
                  layer_norm_eps=1e-5 if family == "clip" else 1e-6)
    if family == "clip":
        vision["hidden_act"] = "quick_gelu"
        cfg = tr.CLIPConfig(text_config=to.clip_text_config("micro").to_dict(), vision_config=vision, projection_dim=96)
        model = init_model(tr.CLIPModel, cfg, 1, norms=("layer_norm", "layrnorm"), f32=("position_embedding",))
    else:
        vision["hidden_act"] = "gelu_pytorch_tanh"
        cfg = tr.SiglipConfig(text_config=to.siglip_text_config().to_dict(), vision_config=vision)
        cfg._attn_implementation = "eager"
        model = init_model(tr.SiglipModel, cfg, 1, norms=("norm",), f32=("position_embedding", "probe"))
    with torch.no_grad():
        model.logit_scale.fill_(np.log(10.0))
    model.save_pretrained(str(tmp_path))
    st, cj = str(tmp_path / "model.safetensors"), str(tmp_path / "config.json")
    pkg.convert.main([st, str(tmp_path / "img.gguf"), "--hf-config", cj])
    pkg.convert.main([st, str(tmp_path / "txt.gguf"), "--hf-config", cj, "--text"])
    mi = eng.vit_model_load(str(tmp_path / "img.gguf"), 0, 8)
    mt = eng.vit_model_load(str(tmp_path / "txt.gguf"), 0, 8)
    imgs = gf.synthetic_images(4, 64, seed=2) * 0.5
    vf = gf.read_gguf(str(tmp_path / "txt.gguf"))
    ids = _ids(family, vf, B=5)
    _, _, _, img_emb = eng.vit_predict(mi, imgs, topk=1, want_logits=True)
    txt_emb, _ = eng.vit_encode_text(mt, ids)
    ta = mt.text_arch
    got = eng.zero_shot_logits(img_emb, txt_emb, ta["logit_scale"], ta["logit_bias"])
    m = model.double()
    with torch.no_grad():
        out = m(input_ids=torch.from_numpy(ids.astype(np.int64)), pixel_values=torch.from_numpy(imgs.transpose(0, 3, 1, 2).astype(np.float64)))
    ref = out.logits_per_image.numpy()
    print(family, "zero-shot max |diff|", np.abs(got - ref).max(), "range", np.ptp(ref))
    assert np.abs(got - ref).max() <= 2e-2 * np.abs(ref).max() + 1e-3
    assert (got.argmax(1) == ref.argmax(1)).all()
    mi.close()
    mt.close()


def test_engine_kinds(towers):
    _, path, _ = towers["siglip"]
    mt = eng.vit_model_load(path, 0, 2)
    x = np.zeros(16, np.float32)
    with pytest.raises(eng.VitB200Error, match="this is a text engine"):
        eng._check(eng.lib().vitb200_forward(mt.handle, x.ctypes.data, 1, x.ctypes.data, None, None, None, 0), "vitb200_forward")
    with pytest.raises(eng.VitB200Error, match="this is a text engine"):
        lib = eng.lib()
        eng._check(lib.vitb200_get_arch(mt.handle, C.byref(eng.Arch())), "vitb200_get_arch")
    with pytest.raises(eng.VitB200Error, match="this is a text engine"):
        mt.set_image_proc(None)
    from tests.util import model_path
    mi = eng.vit_model_load(model_path("micro", "f16"), 0, 2)
    assert mi.text_arch is None
    with pytest.raises(eng.VitB200Error, match="this is an image engine"):
        eng._check(eng.lib().vitb200_encode_text(mi.handle, np.zeros(16, np.int32).ctypes.data, 1, np.zeros(96, np.float32).ctypes.data,
                                                 None, None), "vitb200_encode_text")
    mt.close()
    mi.close()
