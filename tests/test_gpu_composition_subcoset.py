"""The composition polynomial from the CE rows of its sub-coset only, as wf_prove_fib / wf_prove_air build it:
- the constraint kernels on the sub-coset of m rows (wf_eval_constraints_fib_subcoset, wf_eval_constraints_subcoset,
  interpreted and compiled) equal rows j * (ce / m) of the whole-domain evaluation, with every row-keyed input of
  constraint_descs.py (periodic columns, sequence assertions, exemptions, aux segment, ce_blowup 2 to 128);
- wf_composition_commit on those n rows (one column: its coefficients are the interpolation's output, and coset 0 of the LDE
  is the n rows themselves) equals the whole-domain path and a full wf_mat_lde of the same coefficients, on random words,
  i.e. on constraint evaluations that are not those of a low-degree polynomial;
- proofs of traces with one changed cell reproduce tests/golden/invalid_proof_digests.json."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

import constraint_descs as CD
import trace_validate_ref as TV
import winterfell_b200 as wf

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_invalid_proof_digests as golden  # noqa: E402

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    assert c.mem_stats()[0] == 0, "device buffers left live"
    c.close()


def subcoset_sizes(n, ce):
    """m = n (the prover's sub-coset when kc = 1), m = ce (the whole domain, step 1), and the smallest and largest others"""
    return sorted({n, ce, max(1, n // 4), ce // 2} - {0})


# ---- FibSmall kernel ----
@pytest.mark.parametrize("k,log_n,blowup,ext", [
    (1, 3, 2, 1), (1, 9, 8, 3), (2, 4, 16, 2), (5, 6, 8, 2), (32, 5, 8, 3), (4, 12, 4, 1), (3, 14, 2, 3),
])
def test_fib_subcoset_rows(ctx, k, log_n, blowup, ext):
    rng = np.random.default_rng(k * 100 + log_n)
    live0 = ctx.mem_stats()[0]
    n = 1 << log_n
    ce = 2 * n
    results = [int(v) for v in CD.draw(k, rng)]
    lde = ctx.mat_from_host_columns(CD.draw((n * blowup, 2 * k), rng).T)
    coeffs = CD.draw((5 * k, ext), rng)
    full_m = ctx.eval_constraints_fib(k, results, log_n, blowup, ext, lde, coeffs)
    full = full_m.to_rows()
    full_m.free()
    for m in subcoset_sizes(n, ce):
        out = ctx.eval_constraints_fib_subcoset(k, results, log_n, blowup, ext, lde, coeffs, m)
        assert out.rows == m
        assert np.array_equal(out.to_rows(), full[:: ce // m]), m
        out.free()
    lde.free()
    assert ctx.mem_stats()[0] == live0


# ---- generic kernel, interpreted and compiled ----
def run_generic(ctx, desc, log_n, blowup, ext, seed):
    rng = np.random.default_rng(seed)
    live0 = ctx.mem_stats()[0]
    A = TV.Air(desc)
    n = 1 << log_n
    ce = n << A.log_ce_blowup()
    N = n * blowup
    m_lde = ctx.mat_from_host_columns(CD.draw((N, A.w), rng).T)
    a_lde = ctx.mat_from_host_columns(CD.draw((N, A.aw * ext), rng).T) if A.aw else None
    ncc = len(A.degrees) + len(A.aux_degrees) + len(A.asserts) + len(A.aux_asserts)
    coeffs = CD.draw((ncc, ext), rng)
    rand = CD.draw((A.nr, ext), rng) if A.aw else None
    for jit in (True, False):
        ctx.set_jit(jit)
        s0 = ctx.jit_stats()
        full_m = ctx.eval_constraints(desc, log_n, blowup, ext, m_lde, a_lde, coeffs, rand)
        full = full_m.to_rows()
        full_m.free()
        for m in subcoset_sizes(n, ce):
            out = ctx.eval_constraints_subcoset(desc, log_n, blowup, ext, m_lde, a_lde, coeffs, rand, m)
            assert out.rows == m
            assert np.array_equal(out.to_rows(), full[:: ce // m]), (jit, m)
            out.free()
        s1 = ctx.jit_stats()
        assert s1["fallbacks"] == s0["fallbacks"], "the JIT fell back to the interpreter"
        ran = (s1["compiled"] + s1["cache_hits"]) - (s0["compiled"] + s0["cache_hits"])
        assert (ran > 0) == jit, s1
    ctx.set_jit(True)
    for mat in (m_lde, a_lde):
        if mat is not None:
            mat.free()
    assert ctx.mem_stats()[0] == live0


@pytest.mark.parametrize("groups", [4, 9])
def test_boundary_groups_subcoset(ctx, groups):
    """single, periodic and sequence assertions (sequence tables keyed on the CE row, shifts that wrap)"""
    for log_n, blowup, ext in ((4, 8, 1), (7, 4, 3), (10, 2, 2)):
        run_generic(ctx, CD.boundary_groups(1 << log_n, groups, np.random.default_rng(groups)), log_n, blowup, ext, seed=groups + log_n)


@pytest.mark.parametrize("groups", [1, 9])
def test_aux_groups_subcoset(ctx, groups):
    for log_n, blowup, ext in ((4, 4, 1), (6, 8, 2), (9, 4, 3)):
        run_generic(ctx, CD.aux_groups(1 << log_n, groups, np.random.default_rng(groups)), log_n, blowup, ext, seed=groups + log_n)


@pytest.mark.parametrize("count", [1, 8])
def test_exemptions_subcoset(ctx, count):
    for log_n, blowup, ext in ((4, 4, 3), (8, 8, 1)):
        run_generic(ctx, CD.exemptions(1 << log_n, count, np.random.default_rng(count)), log_n, blowup, ext, seed=count)


def test_periodic_columns_subcoset(ctx):
    for log_n, blowup, ext in ((3, 4, 2), (6, 8, 3), (11, 4, 1)):
        run_generic(ctx, CD.periodic(1 << log_n, np.random.default_rng(log_n)), log_n, blowup, ext, seed=log_n)


@pytest.mark.parametrize("ceb", [2, 4, 8, 16, 32, 64, 128])
def test_ce_blowup_subcoset(ctx, ceb):
    log_n = 4 if ceb >= 64 else 6
    ext = (1, 2, 3)[ceb.bit_length() % 3]
    desc = CD.ce_blowup(1 << log_n, ceb, np.random.default_rng(ceb))
    for blowup in (ceb, 2 * ceb) if ceb < 128 else (ceb,):
        run_generic(ctx, desc, log_n, blowup, ext, seed=ceb + blowup)


def test_subcoset_refusals(ctx):
    n, log_n, blowup = 64, 6, 4
    live0 = ctx.mem_stats()[0]
    desc = CD.boundary_groups(n, 3, np.random.default_rng(0))
    A = TV.Air(desc)
    cf = np.zeros((len(A.degrees) + len(A.asserts), 2), dtype=np.uint64)
    lde = ctx.mat_from_host_columns(np.zeros((A.w, n * blowup), dtype=np.uint64))
    flde = ctx.mat_from_host_columns(np.zeros((4, n * blowup), dtype=np.uint64))
    fc = np.zeros((10, 2), dtype=np.uint64)
    for rows in (0, 3, 96, 4 * n):   # empty, not a power of two, larger than the CE domain (ce = 2n)
        with pytest.raises(wf.WfError):
            ctx.eval_constraints_subcoset(desc, log_n, blowup, 2, lde, None, cf, None, rows)
        with pytest.raises(wf.WfError):
            ctx.eval_constraints_fib_subcoset(2, [1, 2], log_n, blowup, 2, flde, fc, rows)
        assert ctx.mem_stats()[0] == live0 + 2
    lde.free()
    flde.free()
    assert ctx.mem_stats()[0] == live0


# ---- composition polynomial and its LDE from the n sub-coset rows ----
@pytest.mark.parametrize("log_n,blowup,ext", [(log_n, blowup, ext) for log_n, blowup in ((3, 2), (6, 128), (11, 8), (12, 8), (16, 4))
                                               for ext in (1, 2, 3)] + [(23, 2, 1)])
def test_composition_lde_reuses_coset0(ctx, log_n, blowup, ext):
    """one column from n rows: the LDE equals wf_mat_lde of the coefficients, its coset 0 is the rows given, and the commitment
    is that of the full LDE (log_n 3, 6, 11: one-pass transforms; 12, 16: two passes; 23: three passes)"""
    rng = np.random.default_rng(log_n * 10 + ext)
    live0 = ctx.mem_stats()[0]
    n = 1 << log_n
    rows = CD.draw((n, ext), rng)
    comp = ctx.mat_from_host_columns(np.ascontiguousarray(rows.T))
    polys, lde, tree = ctx.composition_commit(wf.HASH_BLAKE3_256, comp, log_n, blowup, ext, 1)
    want_polys = comp.interpolate_with_offset(7)
    want_lde = want_polys.lde(blowup.bit_length() - 1)
    want_tree = ctx.commit_rows(wf.HASH_BLAKE3_256, want_lde)
    got_lde = lde.to_rows()
    assert np.array_equal(polys.to_rows(), want_polys.to_rows())
    assert np.array_equal(got_lde, want_lde.to_rows())
    assert np.array_equal(got_lde[::blowup], rows)
    assert tree.root() == want_tree.root()
    for o in (comp, polys, lde, tree, want_polys, want_lde, want_tree):
        o.free()
    assert ctx.mem_stats()[0] == live0


@pytest.mark.parametrize("k,log_n,blowup,ext", [(1, 6, 8, 1), (4, 10, 8, 3), (32, 9, 8, 3), (2, 12, 16, 2)])
def test_fib_composition_equals_whole_domain_path(ctx, k, log_n, blowup, ext):
    """random frames (the evaluations of no low-degree polynomial): the composition commitment from the n sub-coset rows equals
    the one from the whole CE domain"""
    rng = np.random.default_rng(k + log_n)
    live0 = ctx.mem_stats()[0]
    n = 1 << log_n
    results = [int(v) for v in CD.draw(k, rng)]
    lde = ctx.mat_from_host_columns(CD.draw((n * blowup, 2 * k), rng).T)
    coeffs = CD.draw((5 * k, ext), rng)
    full = ctx.eval_constraints_fib(k, results, log_n, blowup, ext, lde, coeffs)
    sub = ctx.eval_constraints_fib_subcoset(k, results, log_n, blowup, ext, lde, coeffs, n)
    a = ctx.composition_commit(wf.HASH_BLAKE3_256, full, log_n, blowup, ext, 1)
    b = ctx.composition_commit(wf.HASH_BLAKE3_256, sub, log_n, blowup, ext, 1)
    assert np.array_equal(a[0].to_rows(), b[0].to_rows())
    assert np.array_equal(a[1].to_rows(), b[1].to_rows())
    assert a[2].root() == b[2].root()
    for o in (lde, full, sub) + a + b:
        o.free()
    assert ctx.mem_stats()[0] == live0


# ---- whole proofs of traces that do not satisfy their AIR ----
@pytest.mark.parametrize("idx", range(len(golden.CASES)))
def test_invalid_trace_proofs_reproduce_golden_digests(ctx, idx):
    with open(os.path.join(HERE, "golden", "invalid_proof_digests.json")) as f:
        rec = json.load(f)[idx]
    case = golden.CASES[idx]
    assert [rec["kind"], rec["name"], rec["log_n"], rec["opts"], rec["cell"]] == [case[0], case[1], case[2], case[3], list(case[4])]
    proof = golden.prove(ctx, case)
    assert len(proof) == rec["bytes"] and hashlib.sha256(proof).hexdigest() == rec["sha256"]
