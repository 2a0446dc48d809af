"""The persistent split-precision attention (attention_wgmma_persistent_kernel, N <= 200, not causal) against the one-CTA-per-(image,
head) kernel it replaces there, bit for bit: at token counts on both sides of its limit (201 and 224 must run the per-head kernel), at
problem counts that leave the CTAs of the persistent grid uneven work, and with a NaN in one image, which must stay in that image.
The hooks fill their output with NaN first, so a row a kernel never writes fails too."""
import numpy as np
import pytest

from tests.util import pkg

eng = pkg.engine
pytestmark = pytest.mark.gpu


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _qkv(B, N, H, seed):
    return np.random.default_rng(seed).standard_normal((B * N, 3 * H * 64)).astype(np.float32)


def _both(qkv, B, N, H):
    new = eng.test_attention_hd(qkv, B, N, H, 64, split=True, kernel=eng.ATTN_WGMMA)
    old = eng.test_attention_hd(qkv, B, N, H, 64, split=True, kernel=eng.ATTN_WGMMA_HEAD)
    return new, old


def _assert_bits_equal(new, old):
    bad = np.argwhere(new.view(np.uint32) != old.view(np.uint32))
    assert bad.size == 0, (len(bad), bad[:5].tolist())


@pytest.mark.parametrize("N", [1, 17, 196, 197, 200, 201, 224])
def test_matches_per_head_kernel_at_token_counts(N):
    B, H = 3, 12
    new, old = _both(_qkv(B, N, H, seed=N), B, N, H)
    assert np.isfinite(old).all()
    _assert_bits_equal(new, old)


@pytest.mark.parametrize("problems", ["below", "equal", "k_plus_1"])
def test_matches_per_head_kernel_at_uneven_problem_counts(problems):
    """B H below the SM count (idle CTAs), equal to it (one problem each) and 2 num_sms + 1 (one CTA takes a third problem)."""
    sms = _num_sms()
    N, H = 197, 1
    B = {"below": sms // 2, "equal": sms, "k_plus_1": 2 * sms + 1}[problems]
    new, old = _both(_qkv(B, N, H, seed=B), B, N, H)
    assert np.isfinite(old).all()
    _assert_bits_equal(new, old)


@pytest.mark.parametrize("N", [17, 197])
def test_nan_stays_in_its_image(N):
    B, H = 5, 12
    qkv = _qkv(B, N, H, seed=7)
    bad_img = 2
    qkv[bad_img * N + N // 2, H * 64 + 5] = np.nan  # one key of head 0 of image 2
    qkv[bad_img * N + 1, 2 * H * 64 + 70] = np.nan  # one value of head 1 of image 2
    new, old = _both(qkv, B, N, H)
    rows = np.arange(B * N) // N
    assert np.isfinite(new[rows != bad_img]).all()
    assert np.isnan(new[rows == bad_img]).any()
    assert (np.isnan(new) == np.isnan(old)).all()
    fin = ~np.isnan(old)
    _assert_bits_equal(new[fin], old[fin])
