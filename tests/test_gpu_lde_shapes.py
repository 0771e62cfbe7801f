"""LDE shapes of the two-pass schedule (n >= 2^12) that the parity tests do not reach: one-column matrices (segment width 1,
where a lane pair of the strided pass spans two tile columns), and column counts that leave the last segment partly
filled. Bit-exact against the CPU oracle."""
import pytest

import winterfell_b200 as wf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("log_n,cols,log_b", [(12, 1, 3), (13, 1, 2), (15, 1, 1), (12, 2, 2), (14, 5, 3), (12, 9, 3)])
def test_two_pass_lde_narrow_and_partial_segments(ctx, oracle, log_n, cols, log_b):
    n = 1 << log_n
    polys = oracle.rand_elems((cols, n), 300 + 10 * log_n + cols)
    want = oracle.lde_rows(polys, 1 << log_b)
    m = ctx.mat_from_host_columns(polys)
    lde = m.lde(log_b)
    assert (lde.to_rows() == want).all()
    into = ctx.mat_from_host_columns(oracle.rand_elems((cols, n << log_b), 5))   # random words, overwritten by lde_into
    m.lde_into(log_b, into)
    assert (into.to_rows() == want).all()
    m.free(); lde.free(); into.free()
