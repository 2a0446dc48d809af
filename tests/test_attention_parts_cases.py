"""CPU checks of the cases of tests/test_gpu_attention_parts.py (built in tests/attention_parts.py).  A float64 model of the kernels'
product set, S = Ql Kh^T + Qh Kl^T + Qh Kh^T and O = P Vl + P Vh, must give each case's expected output exactly.  The same model with
the tested product removed, or with its lo operand read from column group 0 or from row 0, must differ from it in at least one row of
every (image, head).  So each GPU case can tell a kernel that drops or misplaces the product from a correct one."""
import numpy as np
import pytest

from tests import attention_parts as ap
from tests.test_gpu_kernels import _attention_ref
from tests.util import pkg

eng = pkg.engine


def _check_design(f, ops, want, product, c=None):
    assert np.array_equal(ap.model(f, ops), want)
    # no case has a Ql Kl product, so the reference attention on hi + lo computes the same thing
    hi, lo = ap.pack(ops)
    N = want.shape[1]
    ref = _attention_ref(hi.astype(np.float64) + lo.astype(np.float64), ap.B, N, f.H, f.hd, f.causal)
    assert np.array_equal(ref.astype(np.float16).astype(np.float32).reshape(want.shape), want)
    broken = {"dropped": ap.model(f, ops, tuple(p for p in ap.PRODUCTS if p != product))}
    broken.update({name: ap.model(f, m) for name, m in ap.misplaced(ops, product, c).items()})
    expected = {"dropped"} | ({"group 0"} if c != 0 else set()) | ({"row 0"} if N > 1 else set())
    assert set(broken) == expected
    for name, out in broken.items():
        caught = (out != want).any(axis=-1).any(axis=1)        # [B][H]: some row of the (image, head) differs
        assert caught.all(), (name, np.argwhere(~caught).tolist())


@pytest.mark.parametrize("form,N,product", sorted({(form, n, p) for form, n, p, _ in ap.GROUP_CASES}))
def test_score_product_cases_tell_a_broken_product(form, N, product):
    f = ap.FORMS[form]
    for c in range(0, f.hd, ap.GROUP):
        ops, want = ap.group_case(f, N, product, c)
        _check_design(f, ops, want, product, c)


@pytest.mark.parametrize("form,N", ap.PVL_CASES, ids=ap.PVL_IDS)
def test_p_vl_cases_tell_a_broken_product(form, N):
    f = ap.FORMS[form]
    ops, want = ap.pvl_case(f, N)
    _check_design(f, ops, want, "PVl")
    if N == 1:  # one key: its lo(v) row only, which dropping P Vl turns to 0
        assert (want != 0).any(axis=-1).all()


def test_every_form_and_group_is_covered():
    """8 column groups at head dim 64, 10 at 80, 9 at 72, each for both score products at three token counts; P Vl at every N."""
    groups = {form: len({c for fm, _, _, c in ap.GROUP_CASES if fm == form}) for form in ap.FORMS}
    assert groups == {"wgmma": 8, "causal": 8, "hd80split": 10, "hd72split": 9}
    assert len(ap.GROUP_CASES) == 2 * 3 * sum(groups.values())
    assert len(ap.PVL_CASES) == 4 * 7


@pytest.mark.parametrize("hd", [80, 72])
def test_parts_hook_runs_the_causal_mask_at_head_dim_64_only(hd):
    z = np.zeros((ap.B * 4, 3 * hd), np.float16)
    with pytest.raises(ValueError, match=f"head dim 64 only, not {hd}"):
        eng.test_attention_parts(z, z, ap.B, 4, 1, hd, causal=True)


def test_parts_hook_refuses_other_head_dims():
    z = np.zeros((4, 3 * 96), np.float16)
    with pytest.raises(ValueError, match="head dims 64, 80 and 72, not 96"):
        eng.test_attention_parts(z, z, 1, 4, 1, 96)
