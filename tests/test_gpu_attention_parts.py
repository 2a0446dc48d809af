"""Each lo-half product of the split-precision attention alone, bit for bit: Ql Kh^T and Qh Kl^T on every 8-column group, and P Vl on
every key, in the head-dim-64 wgmma kernel (plain and causal) and the row-major kernel at head dims 80 and 72.  The operands lie in one
half only (tests/attention_parts.py), so every probability row is one-hot only when the product under test reads the right columns and
keys.  The hooks fill their output with NaN first, so a row a kernel never writes fails too."""
import numpy as np
import pytest

from tests import attention_parts as ap

pytestmark = pytest.mark.gpu


def _assert_routed(f, ops, want):
    got = ap.run(f, ops)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (len(bad), bad[:5].tolist())


@pytest.mark.parametrize("form,N,product,c", ap.GROUP_CASES, ids=ap.GROUP_IDS)
def test_score_product_alone_routes_every_row(form, N, product, c):
    """Qh Kl (q in hi, the key patterns in lo(k)) or Ql Kh (q in lo, the patterns in hi(k)) on columns [c, c + 8) is the only
    non-zero score: output row i must be v of its chosen key.  A product dropped, stepped through the columns wrongly or fed half a
    fragment leaves the scores flat (the mean of v) or routes rows to another key."""
    f = ap.FORMS[form]
    _assert_routed(f, *ap.group_case(f, N, product, c))


@pytest.mark.parametrize("form,N", ap.PVL_CASES, ids=ap.PVL_IDS)
def test_p_vl_alone_routes_every_row(form, N):
    """One-hot rows through Qh Kh, hi(v) = 0: output row i must be lo(v) of its chosen key.  Every key is some row's choice, so a lo V
    tile dropped or read at another key step or n8 column tile changes some row."""
    f = ap.FORMS[form]
    _assert_routed(f, *ap.pvl_case(f, N))
