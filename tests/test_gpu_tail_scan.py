"""The synthetic division of the coefficient-form DEEP composition (syn_div_reduce / _carry / _apply) at the sizes where its scan
changes shape, and the FRI commit phase at the lengths where the layer loop changes shape.

The division keeps, per thread, the run of the lanes above it in its warp and, per warp, the run of the warps above it in its
tile (2048 rows = 8 warps x 32 lanes x 8 rows), and combines runs by powers of z read from a table. n = 8 and 2^8 leave most
lanes or warps of the one tile empty, 2^11 fills exactly one tile, 2^12 and 2^13 carry over two and four tiles. Each case is
checked against the reference's serial syn_div (polynom/mod.rs:498-505) run on the host, for z random, z = p - 1 (powers
alternate in sign) and z = 1 (every power is 1).

FRI: a codeword of exactly (remainder bound) x folding points commits one layer whose fold writes the remainder, and one of
(remainder bound) points commits none; both against the oracle's FriProver, for every folding factor and extension degree (the
cubic codeword is stored with a zero pad lane, which the fold writes itself)."""
import numpy as np
import pytest

import combine_model as M
import winterfell_b200 as wf

P = wf.P


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def _zg(oracle, z, log_n):
    g = oracle.root_of_unity(log_n)
    return np.array([oracle.mul(int(v), g) for v in z], dtype=np.uint64)


@pytest.mark.gpu
@pytest.mark.parametrize("ext,log_n", [(1, 3), (3, 3), (2, 8), (3, 8), (1, 11), (2, 11), (3, 11), (3, 12), (2, 13)])
@pytest.mark.parametrize("zkind", ["random", "p - 1", "1"])
def test_division_matches_serial_syn_div_at_tile_shapes(ctx, oracle, ext, log_n, zkind):
    n, c, kc = 1 << log_n, 3, 1
    main_cols = oracle.rand_elems((c, n), 300 + log_n * 7 + ext)
    cons_cols = oracle.rand_elems((kc, n * ext), 400 + log_n * 7 + ext)
    coeffs = oracle.rand_elems((c + kc, ext), 500 + ext)
    z = {"random": oracle.rand_elems((ext,), 600 + log_n), "p - 1": np.array([P - 1] + [0] * (ext - 1), dtype=np.uint64),
         "1": np.array([1] + [0] * (ext - 1), dtype=np.uint64)}[zkind]
    main = ctx.mat_from_host_columns(main_cols)
    cons = ctx.mat_from_host_columns(cons_cols, ext_degree=ext)
    deep = ctx.deep_compose_polys(ext, main, None, cons, 1, z, coeffs)
    coef = deep.interpolate_with_offset(7).to_rows()   # the quotient's coefficients, 2n rows
    S = np.zeros((n, ext), dtype=np.uint64)
    for j in range(c):
        t = M.np_ext_mul(np.stack([main_cols[j]] + [np.zeros(n, dtype=np.uint64)] * (ext - 1), axis=1), coeffs[j:j + 1])
        S = np.stack([(S[:, q].astype(object) + t[:, q].astype(object)) % P for q in range(ext)], axis=1).astype(np.uint64)
    t = M.np_ext_mul(cons_cols[0].reshape(n, ext), coeffs[c:c + 1])
    S = np.stack([(S[:, q].astype(object) + t[:, q].astype(object)) % P for q in range(ext)], axis=1).astype(np.uint64)
    qz, qzg = M.host_syn_div(oracle, S, z, ext), M.host_syn_div(oracle, S, _zg(oracle, z, log_n), ext)
    want = ((qz.astype(object) + qzg.astype(object)) % P).astype(np.uint64)
    assert np.array_equal(coef[:n], want)
    assert not coef[n:].any()
    for o in (main, cons, deep):
        o.free()


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("nf", [2, 4, 8, 16])
@pytest.mark.parametrize("layers", [0, 1])
def test_fri_commit_at_the_remainder_bound(ctx, oracle, d, nf, layers):
    rem_max_deg, blowup = 7, 8
    L = (rem_max_deg + 1) * blowup * (nf if layers else 1)
    ev = oracle.rand_elems((1, L * d), 700 + 10 * nf + d)
    m = ctx.mat_from_host_columns(ev, ext_degree=d)
    f, roots = ctx.fri_build_layers_default(wf.HASH_BLAKE3_256, m, d, nf, rem_max_deg, blowup)
    want_roots, want_rem, _ = oracle.fri_build_layers(oracle.BLAKE3, ev[0], nf, rem_max_deg, blowup, d)
    assert f.num_layers == layers
    assert np.array_equal(roots, want_roots)
    assert np.array_equal(f.remainder(), want_rem)
    f.free()
    m.free()
