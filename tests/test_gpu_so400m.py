"""SigLIP So400m-shaped towers on the GPU: the head-dim-72 attention kernel (split and f16 forms) and the 72-column pooling kernel against
float64, and image and text towers end to end against float64 Hugging Face (tests/so400m_oracle.py), each output within twice the
emulation's own distance from it, as tests/test_gpu_siglip.py holds the head-dim-64 towers."""
import numpy as np
import pytest

from tests.util import pkg, gf
from tests import siglip_oracle as sgo
from tests import so400m_oracle as so
from tests import text_oracle as to
from tests import fp8_reference as fr
from tests.hf_oracle import save_and_convert
from tests.test_gpu_fp8 import E2E_TOL

eng = pkg.engine
pytestmark = pytest.mark.gpu

SPLIT_N = [1, 15, 16, 17, 31, 32, 33, 127, 128, 129, 197, 223, 224]
F16_N = [225, 256, 257, 288, 289, 577, 729, 799, 800]


@pytest.mark.parametrize("N", SPLIT_N + F16_N)
def test_attention_kernel_against_float64(N):
    """H = 3 (head slices at 0, 144 and 288 B), B = 2; split precision up to 224 tokens, f16 operands beyond.  A NaN in image 1's k
    leaves image 0 bit-identical; uniform scores give each image's plain mean of v."""
    B, H, hd = 2, 3, 72
    split = N <= 224
    rng = np.random.default_rng(N)
    qkv = rng.standard_normal((B * N, 3 * H * hd)).astype(np.float32)
    if not split:
        qkv = qkv.astype(np.float16).astype(np.float32)
    out = eng.test_attention_hd72(qkv, B, N, H, split)
    want = so.attention_ref(qkv, B, N, H, hd)
    err = np.abs(out - want).max()
    assert err <= (2e-3 if split else 4e-3) * np.abs(want).max() + 1e-3, err
    bad = qkv.copy()
    bad[N + N // 2, H * hd + 7] = np.nan
    got = eng.test_attention_hd72(bad, B, N, H, split)
    assert np.array_equal(got[:N], out[:N])
    uni = qkv.copy()
    uni[:, : 2 * H * hd] = 0.0
    uni[:, 2 * H * hd:] = np.repeat(np.arange(1, B + 1, dtype=np.float32), N)[:, None]
    got = eng.test_attention_hd72(uni, B, N, H, split)
    assert np.array_equal(got, np.repeat(np.arange(1, B + 1, dtype=np.float32), N)[:, None] * np.ones((1, H * hd), np.float32))


def test_attention_hook_limits():
    qkv = np.zeros((801, 3 * 72), np.float32)
    with pytest.raises(eng.VitB200Error, match="801 tokens not supported \\(max 800 at head dim 72"):
        eng.test_attention_hd72(qkv, 1, 801, 1, False)
    with pytest.raises(eng.VitB200Error, match="split-precision head-dim-72 attention needs N <= 224"):
        eng.test_attention_hd72(qkv[:225], 1, 225, 1, True)


@pytest.mark.parametrize("P", [1, 16, 256, 729, 800])
def test_attention_pool_kernel_against_float64(P):
    """Random q, k, v (row-major [B*P][2 D]) against float64; a NaN in image 1's k or v leaves the others bit-identical; uniform scores
    give each image's mean."""
    B, H, hd = 3, 2, 72
    D = H * hd
    rng = np.random.default_rng(P)
    q = rng.standard_normal(D).astype(np.float32)
    kv = rng.standard_normal((B * P, 2 * D)).astype(np.float16)
    out = eng.test_attention_pool_hd72(q, kv, B, P, H)
    want = so.pool_ref(q, kv, B, P, H)
    assert np.abs(out - want).max() <= 2e-3 * np.abs(want).max() + 1e-3, np.abs(out - want).max()
    for col in (3, 70, D + 5, D + 71):
        bad = kv.copy()
        bad[P + P // 2, col] = np.nan
        got = eng.test_attention_pool_hd72(q, bad, B, P, H)
        assert np.array_equal(got[0], out[0]) and np.array_equal(got[2], out[2]), col
    uni = np.zeros((B * P, 2 * D), np.float16)
    for b in range(B):
        uni[b * P:(b + 1) * P, D:] = b + 1
    got = eng.test_attention_pool_hd72(q, uni, B, P, H)
    assert np.array_equal(got, np.repeat(np.arange(1, B + 1, dtype=np.float32), D).reshape(B, D))


_built = {}


def _case(geo, classifier, tmp_path_factory):
    key = (geo, classifier)
    if key not in _built:
        d = str(tmp_path_factory.mktemp(f"{geo}_{classifier}"))
        m = so.build_hf(geo, classifier)
        path = save_and_convert(m, d, "siglip")
        vf = gf.read_gguf(path)
        imgs = gf.synthetic_images(3, vf.img_size, seed=3)
        o = sgo.hf_outputs(m, imgs)
        emu = so.Emulation(vf, acc=np.float64, fp8=False)
        L = vf.num_hidden_layers
        x = {i: emu.encode(imgs, i) for i in (0, L - 1, L)}
        emu_d = {"logits": fr.rel_dist(emu.forward(imgs), o["logits"]), "prelogits": fr.rel_dist(emu.prelogits(x[L]), o["prelogits"]),
                 "last_hidden_state": fr.rel_dist(emu.final_ln(x[L]), o["last_hidden_state"])}
        emu_d.update({f"tokens{i}": fr.rel_dist(x[i], o["hidden_states"][i]) for i in x})
        _built[key] = (path, vf, imgs, o, emu_d)
    return _built[key]


CASES = [(g, c) for g in so.GEOMETRIES for c in (False, True)]


@pytest.mark.parametrize("geo,classifier", CASES, ids=[f"{g}-{'cls' if c else 'model'}" for g, c in CASES])
def test_end_to_end_against_the_hf_oracle(geo, classifier, tmp_path_factory):
    """logits, prelogits, last_hidden_state, hidden_states[0, L-1, L] and the embed tap, each within twice the emulation's distance."""
    path, vf, imgs, o, emu_d = _case(geo, classifier, tmp_path_factory)
    L, n, D, P = vf.num_hidden_layers, imgs.shape[0], vf.hidden_size, vf.n_tokens
    m = eng.vit_model_load(path, 0, n)
    assert m.pool == ("mean" if classifier else "map") and m.n_tokens == P == (vf.img_size // vf.patch_size) ** 2
    assert m.mlp_dim == so.GEOMETRIES[geo][2]
    _, _, _, logits = eng.vit_predict(m, imgs, 5, want_logits=True)
    got = {"logits": fr.rel_dist(logits, o["logits"])}
    tok, pre = eng.vit_features(m, imgs, layers=L, norm=True, prelogits=True)
    got["prelogits"] = fr.rel_dist(pre.reshape(n, -1), o["prelogits"])
    got["last_hidden_state"] = fr.rel_dist(tok, o["last_hidden_state"])
    for i in (0, L - 1, L):
        tok, _ = eng.vit_features(m, imgs, layers=i, norm=False)
        got[f"tokens{i}"] = fr.rel_dist(tok, o["hidden_states"][i])
    _, _, taps = eng.vit_predict_debug(m, imgs, 0, taps=("embed", "h"))
    assert taps["h"].shape == (n, P, m.mlp_dim)
    got["embed"] = fr.rel_dist(taps["embed"], o["hidden_states"][0])
    emu_d["embed"] = emu_d["tokens0"]
    m.close()
    print(geo, classifier, {k: f"{got[k].max():.2e} (emulation {emu_d[k].max():.2e})" for k in got})
    bad = {k: (got[k].max(), emu_d[k].max()) for k in got if got[k].max() > 2 * emu_d[k].max()}
    assert not bad, bad


@pytest.mark.parametrize("geo", ["micro72_p14", "so400m_224", "so400m_384"])
def test_launch_count_batch_invariance_graphs_and_isolation(geo, tmp_path_factory):
    """2 + 7 L + 10 launches (map) and 2 + 7 L + 3 (mean); each image alone, eager and graph-replayed, gives its batch logits bit for bit;
    a NaN pixel inside the grid, a NaN in the dropped border or every pixel at 1e6 in image 1 leaves images 0 and 2 bit for bit, and a
    NaN in the dropped border alone changes no output of image 1 either."""
    for classifier in (False, True):
        p, vf, imgs, _, _ = _case(geo, classifier, tmp_path_factory)
        L = vf.num_hidden_layers
        want = 2 + 7 * L + (3 if classifier else 10)
        m = eng.vit_model_load(p, 0, 3)
        clean = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
        assert m.last_launch_count() == want
        ctok, cpre = eng.vit_features(m, imgs, norm=True, prelogits=True)
        for b in range(3):
            for rep in range(3):
                assert np.array_equal(eng.vit_predict(m, imgs[b:b + 1], 5, want_logits=True)[3][0], clean[b]), (b, rep)
        cut = vf.img_size // vf.patch_size * vf.patch_size
        poisons = {"nan": (1, 5, 7), "big": None}
        if cut < vf.img_size:
            poisons["border"] = (1, vf.img_size - 1, 3)
        for name, at in poisons.items():
            bad = imgs.copy()
            if at is None:
                bad[1] = 1e6
            else:
                bad[at[0], at[1], at[2], 1] = np.nan
                if name == "border":
                    bad[1, 2, vf.img_size - 1, 0] = np.nan
            logits = eng.vit_predict(m, bad, 5, want_logits=True)[3]
            tok, pre = eng.vit_features(m, bad, norm=True, prelogits=True)
            for b in ((0, 1, 2) if name == "border" else (0, 2)):
                assert np.array_equal(logits[b], clean[b]) and np.array_equal(tok[b], ctok[b]) and np.array_equal(pre[b], cpre[b]), (name, b)
        assert np.array_equal(eng.vit_predict(m, imgs, 5, want_logits=True)[3], clean)
        m.close()


def test_profile_kinds_count_the_new_kernels(tmp_path_factory):
    import ctypes as C
    p, vf, imgs, _, _ = _case("so400m_384", False, tmp_path_factory)
    m = eng.vit_model_load(p, 0, 3)
    L = eng.lib()
    eng._check(L.vitb200_profile_enable(m.handle, 1), "profile")
    eng.vit_predict(m, imgs, 5)
    ms, cnt, fl = C.c_double(), C.c_int(), C.c_double()
    eng._check(L.vitb200_profile_read(m.handle, 6, C.byref(ms), C.byref(cnt), C.byref(fl)), "profile_read")
    N, D = vf.n_tokens, vf.hidden_size
    assert cnt.value == vf.num_hidden_layers and fl.value == 4.0 * 3 * N * N * D and ms.value > 0
    eng._check(L.vitb200_profile_read(m.handle, 8, C.byref(ms), C.byref(cnt), C.byref(fl)), "profile_read")
    assert cnt.value == 3 and ms.value > 0
    eng._check(L.vitb200_profile_enable(m.handle, 0), "profile")
    m.close()


def test_every_entry_point_at_384(tmp_path_factory):
    """So400m-384: tensors == file; async, device and sharded forward == vit_predict; the u8 path with vit.cpp's preprocessing and with a
    384 x 384 bicubic SigLIP processor == the f32 path on the images it returns; features from u8 == from f32."""
    import torch
    import ctypes as C
    for classifier in (False, True):
        path, vf, imgs, _, _ = _case("so400m_384", classifier, tmp_path_factory)
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
        torch.cuda.synchronize()
        assert np.array_equal(d_log.cpu().numpy(), ref)
        rng = np.random.default_rng(3)
        u8 = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in ((397, 431), (384, 384), (300, 271))]
        for proc in (None, {"do_resize": True, "size": {"height": 384, "width": 384}, "resample": 3, "do_rescale": True,
                            "rescale_factor": 1 / 255, "do_normalize": True, "image_mean": [0.5] * 3, "image_std": [0.5] * 3}):
            m.set_image_proc(proc)
            f32, _, _, _, logits = eng.vit_image_preprocess_predict(m, u8)
            assert f32.shape == (3, 384, 384, 3)
            assert np.array_equal(logits, eng.vit_predict(m, f32, 5, want_logits=True)[3])
            tok, pre = eng.vit_features_u8(m, u8, layers=1, norm=True, prelogits=True)
            t2, p2 = eng.vit_features(m, f32, layers=1, norm=True, prelogits=True)
            assert np.array_equal(tok, t2) and np.array_equal(pre, p2)
        m.close()


def test_fp8_engine_against_the_fp8_emulation(tmp_path_factory):
    path, vf, imgs, _, _ = _case("micro72", False, tmp_path_factory)
    m = eng.vit_model_load(path, 0, 3, fp8=True)
    logits = eng.vit_predict(m, imgs, 5, want_logits=True)[3]
    m.close()
    d = fr.rel_dist(logits, so.Emulation(vf).forward(imgs))
    assert d.max() <= E2E_TOL, d


def test_text_tower_against_hugging_face(tmp_path):
    """A So400m-shaped SiglipTextModel (D 1152, 16 heads of 72, F 4304): embeds and last_hidden_state within 2e-3 of float64 HF (the
    split-precision attention leaves the f16 roundings of the GEMM operands)."""
    model = so.build_text()
    path = to.convert(model, str(tmp_path))
    vf = gf.read_gguf(path)
    V, N = int(vf.tensors["token_embd.weight"].shape[0]), vf.text["context"]
    ids = to.padded_ids(np.random.default_rng(3), 4, N, V, V - 1, [0, N - 1, 4, None])
    hf = to.hf_outputs(model, ids)
    m = eng.vit_model_load(path, 0, 4)
    assert m.mlp_dim == 4304
    emb, tok = eng.vit_encode_text(m, ids, norm=True, tokens=True)
    m.close()
    d_emb, d_tok = fr.rel_dist(emb, hf["embeds"]).max(), fr.rel_dist(tok, hf["last_hidden_state"]).max()
    print("text", f"{d_emb:.2e} {d_tok:.2e}")
    assert d_emb <= 2e-3 and d_tok <= 2e-3


def test_zero_shot_end_to_end(tmp_path):
    """A SiglipModel with So400m-width towers (so400m_224 and TEXT: D 1152, 16 heads of 72, F 4304): image engine + text engine + the
    sigmoid zero-shot head against HF's logits_per_image, and against zero_shot_logits on the engines' own embeddings."""
    import torch
    model = so.build_clip_pair("so400m_224", seed=1)
    with torch.no_grad():
        model.logit_scale.fill_(np.log(10.0))
    d = str(tmp_path)
    model.save_pretrained(d)
    st, cj = f"{d}/model.safetensors", f"{d}/config.json"
    pkg.convert.main([st, f"{d}/img.gguf", "--hf-config", cj])
    pkg.convert.main([st, f"{d}/txt.gguf", "--hf-config", cj, "--text"])
    tv = gf.read_gguf(f"{d}/txt.gguf")
    V, N = int(tv.tensors["token_embd.weight"].shape[0]), tv.text["context"]
    ids = to.padded_ids(np.random.default_rng(5), 5, N, V, V - 1, [0, N - 1, 4, None, 7])
    imgs = gf.synthetic_images(3, 224, seed=4)
    mt = eng.vit_model_load(f"{d}/txt.gguf", 0, 8)
    temb, _ = eng.vit_encode_text(mt, ids)
    ta = mt.text_arch
    mt.close()
    mi = eng.vit_model_load(f"{d}/img.gguf", 0, 4)
    iemb = eng.vit_predict(mi, imgs, 5, want_logits=True)[3]
    mi.set_zero_shot(temb, logit_scale=ta["logit_scale"], logit_bias=ta["logit_bias"], probs="sigmoid")
    logits = eng.vit_predict(mi, imgs, 5, want_logits=True)[3]
    mi.close()
    host = eng.zero_shot_logits(iemb, temb, ta["logit_scale"], ta["logit_bias"])
    assert np.abs(logits - host).max() <= 1e-4 * np.abs(host).max() + 1e-5
    m = model.double()
    with torch.no_grad():
        out = m(input_ids=torch.from_numpy(ids.astype(np.int64)),
                pixel_values=torch.from_numpy(imgs.astype(np.float64).transpose(0, 3, 1, 2)))
    want = out.logits_per_image.numpy()
    assert np.abs(logits - want).max() <= 2e-2 * np.abs(want).max(), np.abs(logits - want).max()
    assert (logits.argmax(1) == want.argmax(1)).all()
