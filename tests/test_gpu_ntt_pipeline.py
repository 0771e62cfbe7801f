"""NTT pass shapes the parity tests do not reach: launches of many tiles whose count is not a multiple of the SM count,
launches of fewer tiles than there are SMs (2^12 .. 2^16 rows, few columns), one-column segments and partly filled
segments over many tiles, and inverse transforms at each of these shapes. Bit-exact against the CPU oracle."""
import numpy as np
import pytest

import winterfell_b200 as wf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


# (log_n, cols): one pass (n <= 2^11, 300 columns), two passes over many tiles (2^16 .. 2^20, full and partly filled
# 8-wide segments), one-column segments, and 2^12 .. 2^16 with fewer tiles than SMs
SHAPES = [(11, 300), (16, 21), (18, 1), (18, 11), (20, 13), (12, 1), (12, 3), (14, 2), (16, 1)]


@pytest.mark.parametrize("log_n,cols", SHAPES)
def test_forward_and_inverse(ctx, oracle, log_n, cols):
    n = 1 << log_n
    x = oracle.rand_elems((cols, n), 700 + 10 * log_n + cols)
    m = ctx.mat_from_host_columns(x)
    ev = m.evaluate()
    got = ev.to_columns()
    for c in range(cols):
        assert (got[c] == oracle.evaluate_poly(x[c])).all(), (log_n, c)
    back = ev.interpolate()
    assert (back.to_columns() == x).all()
    coefs = m.interpolate()
    assert (np.asarray(coefs.to_columns()) == np.asarray(oracle.interpolate_columns(x))).all()
    m.free(); ev.free(); back.free(); coefs.free()


@pytest.mark.parametrize("log_n,cols,log_b", [(12, 1, 1), (12, 3, 1), (14, 1, 3), (16, 2, 2), (18, 11, 2), (20, 13, 3), (11, 300, 3)])
def test_lde(ctx, oracle, log_n, cols, log_b):
    n = 1 << log_n
    polys = oracle.rand_elems((cols, n), 900 + 10 * log_n + cols)
    m = ctx.mat_from_host_columns(polys)
    lde = m.lde(log_b)
    assert (lde.to_rows() == oracle.lde_rows(polys, 1 << log_b)).all()
    m.free(); lde.free()
