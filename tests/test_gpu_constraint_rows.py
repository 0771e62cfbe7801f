"""The constraint evaluation kernels compared row by row with the oracle (wfo_eval_constraint_rows): the FibSmall kernel
(wf_eval_constraints_fib), the generic kernel interpreted and compiled per AIR (wf_eval_constraints, JIT off and on), and
both over row windows (wf_eval_constraints_window, wf_eval_constraints_fib with row0 / ce_rows) as the row-sharded prover
runs them. LDEs and coefficients are random words with the edge words of constraint_descs.EDGE_WORDS mixed in; the
descriptions of constraint_descs.py are each named for the evaluator path they reach. Shapes up to 2^16 CE rows are
compared on every row, larger ones on sampled rows."""
import ctypes as C
import random

import numpy as np
import pytest

import combine_model as M
import constraint_descs as CD
import trace_validate_ref as TV
import winterfell_b200 as wf
from airs import P

pytestmark = pytest.mark.gpu

FULL_ROWS = 1 << 16


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    assert c.mem_stats()[0] == 0, "device buffers left live"
    c.close()


def sample_rows(ce, rng, extra=(), count=64):
    """rows 0, ce/2 - 1, ce/2 (the twiddle's sign flips), ce - 1 (the next row wraps), `extra` and a random sample"""
    rows = [0, ce // 2 - 1, ce // 2, ce - 1] + [int(r) % ce for r in extra] + [int(r) for r in rng.integers(0, ce, count)]
    return np.unique(np.array(rows, dtype=np.uint64))


def compared_rows(ce, rng):
    return np.arange(ce, dtype=np.uint64) if ce <= FULL_ROWS else sample_rows(ce, rng)


def oracle_rows(oracle, desc, n, blowup, ext, coeffs, rand, rows, lde, alde):
    """the oracle's values on CE rows `rows` from the host LDEs [N, w] and [N, aw * ext]"""
    A = TV.Air(desc)
    shift = (blowup // (1 << A.log_ce_blowup())).bit_length() - 1
    N = n * blowup
    ls = rows.astype(np.int64) << shift
    lx = (ls + blowup) % N
    acur = alde[ls] if A.aw else None
    anxt = alde[lx] if A.aw else None
    return oracle.eval_constraint_rows(desc, n, blowup, ext, coeffs, rand, rows, lde[ls], lde[lx], acur, anxt)


def pad_lane(ctx, mat, ext):
    """the words of the output's segment lanes past `ext` (the output of an extension degree 3 has 4-word rows): the handle's
    first word is the segment base (struct wf_mat { SegMatrix m; }, SegMatrix::base first)"""
    W = 4 if ext == 3 else ext
    if W == ext:
        return np.zeros(0, dtype=np.uint64)
    base = C.cast(mat.h, C.POINTER(C.c_uint64))[0]
    view = ctx.mat_wrap_device(base, mat.rows, W)
    try:
        return view.to_rows()[:, ext:]
    finally:
        view.free()


def eval_generic(ctx, desc, log_n, blowup, ext, m_lde, a_lde, coeffs, rand, jit):
    ctx.set_jit(jit)
    s0 = ctx.jit_stats()
    out = ctx.eval_constraints(desc, log_n, blowup, ext, m_lde, a_lde, coeffs, rand)
    s1 = ctx.jit_stats()
    ctx.set_jit(True)
    assert s1["fallbacks"] == s0["fallbacks"], "the JIT fell back to the interpreter"
    ran = (s1["compiled"] + s1["cache_hits"]) - (s0["compiled"] + s0["cache_hits"])
    assert ran == (1 if jit else 0), s1
    return out


def window_lde(lde, row0, ce_rows, shift, blowup):
    """the LDE rows a window reads: its own rows, then `blowup` halo rows (wrapping to row 0 after the last window)"""
    N = lde.shape[0]
    idx = (np.arange((ce_rows << shift) + blowup) + (row0 << shift)) % N
    return np.ascontiguousarray(lde[idx])


def windows(ce):
    """(row0, ce_rows): the domain cut into 2, 4 and 8 windows, and 64-row windows (all of them up to 16, else the first
    two, two around the middle and the last two)"""
    out = []
    for G in (2, 4, 8):
        if ce // G >= 64:
            out += [(g * (ce // G), ce // G) for g in range(G)]
    starts = list(range(0, ce, 64))
    if len(starts) > 16:
        h = len(starts) // 2
        starts = starts[:2] + starts[h - 1:h + 1] + starts[-2:]
    return out + [(s, 64) for s in starts]


def check_windows(ctx, full, run_window, lde, alde, ce, shift, blowup, ext):
    """every window equals the same rows of the full-domain call; its pad lane is zero"""
    for row0, cr in windows(ce):
        wm = ctx.mat_from_host_columns(window_lde(lde, row0, cr, shift, blowup).T)
        wa = ctx.mat_from_host_columns(window_lde(alde, row0, cr, shift, blowup).T) if alde is not None else None
        out = run_window(wm, wa, row0, cr)
        assert out.rows == cr
        assert np.array_equal(out.to_rows(), full[row0:row0 + cr]), (row0, cr)
        assert not pad_lane(ctx, out, ext).any(), (row0, cr)
        for m in (out, wm, wa):
            if m is not None:
                m.free()


def run_generic(ctx, oracle, desc, log_n, blowup, ext, seed, with_windows=True):
    """desc on a random LDE through the interpreter and the compiled kernel: equal to each other and to the oracle, on
    every window too"""
    rng = np.random.default_rng(seed)
    live0 = ctx.mem_stats()[0]
    A = TV.Air(desc)
    n, ceb = 1 << log_n, 1 << A.log_ce_blowup()
    ce, N, shift = n * ceb, n * blowup, (blowup // ceb).bit_length() - 1
    lde = CD.draw((N, A.w), rng)
    alde = CD.draw((N, A.aw * ext), rng) if A.aw else None
    ncc = len(A.degrees) + len(A.aux_degrees) + len(A.asserts) + len(A.aux_asserts)
    coeffs = CD.draw((ncc, ext), rng)
    rand = CD.draw((A.nr, ext), rng) if A.aw else None
    if A.aw:
        rand[0] = P - 1
    m_lde = ctx.mat_from_host_columns(lde.T)
    a_lde = ctx.mat_from_host_columns(alde.T) if A.aw else None
    outs = [eval_generic(ctx, desc, log_n, blowup, ext, m_lde, a_lde, coeffs, rand, jit) for jit in (True, False)]
    full = outs[0].to_rows()
    assert full.shape == (ce, ext)
    assert np.array_equal(full, outs[1].to_rows()), "compiled and interpreted kernels differ"
    for o in outs:
        assert not pad_lane(ctx, o, ext).any()
        o.free()
    rows = compared_rows(ce, rng)
    want = oracle_rows(oracle, desc, n, blowup, ext, coeffs, rand, rows, lde, alde)
    bad = np.flatnonzero((full[rows.astype(np.int64)] != want).any(axis=1))
    assert bad.size == 0, f"{bad.size} rows differ from the oracle, first CE row {rows[bad[0]]}"
    if with_windows and ce >= 128:
        for jit in (True, False):
            ctx.set_jit(jit)
            check_windows(ctx, full, lambda wm, wa, r0, cr: ctx.eval_constraints_window(desc, log_n, blowup, ext, wm, wa, coeffs, rand,
                                                                                         r0, cr),
                          lde, alde, ce, shift, blowup, ext)
        ctx.set_jit(True)
    for m in (m_lde, a_lde):
        if m is not None:
            m.free()
    assert ctx.mem_stats()[0] == live0
    return full


# ---- FibSmall: the specialised kernel and the generic one on the same coefficients ----
def run_fib(ctx, oracle, k, log_n, blowup, ext, results, seed, lde=None, coeffs=None, windows_too=True):
    rng = np.random.default_rng(seed)
    live0 = ctx.mem_stats()[0]
    n, ce = 1 << log_n, 2 << log_n
    N, shift = n * blowup, (blowup // 2).bit_length() - 1
    lde = CD.draw((N, 2 * k), rng) if lde is None else lde
    coeffs = CD.draw((5 * k, ext), rng) if coeffs is None else coeffs
    desc = CD.fib_desc(k, n, results)
    m = ctx.mat_from_host_columns(lde.T)
    fo = ctx.eval_constraints_fib(k, results, log_n, blowup, ext, m, coeffs)
    fib = fo.to_rows()
    assert not pad_lane(ctx, fo, ext).any()
    fo.free()
    gen = [eval_generic(ctx, desc, log_n, blowup, ext, m, None, coeffs, None, jit) for jit in (True, False)]
    for g in gen:
        assert np.array_equal(g.to_rows(), fib), "the FibSmall and generic kernels differ"
        g.free()
    rows = compared_rows(ce, rng)
    want = oracle_rows(oracle, desc, n, blowup, ext, coeffs, None, rows, lde, None)
    bad = np.flatnonzero((fib[rows.astype(np.int64)] != want).any(axis=1))
    assert bad.size == 0, f"{bad.size} rows differ from the oracle, first CE row {rows[bad[0]]}"
    if windows_too and ce >= 128:
        check_windows(ctx, fib, lambda wm, wa, r0, cr: ctx.eval_constraints_fib(k, results, log_n, blowup, ext, wm, coeffs, r0, cr),
                      lde, None, ce, shift, blowup, ext)
    m.free()
    assert ctx.mem_stats()[0] == live0
    return fib


@pytest.mark.parametrize("k,log_n,blowup,ext", [
    (1, 3, 2, 1), (1, 9, 8, 3), (2, 4, 16, 2), (3, 7, 2, 3), (4, 10, 8, 1), (5, 6, 8, 2),   # k = 5: a partly filled last segment
    (5, 15, 2, 3), (32, 5, 8, 3), (32, 12, 16, 1), (4, 16, 2, 2),
])
def test_fib_kernels_equal_oracle(ctx, oracle, k, log_n, blowup, ext):
    rng = np.random.default_rng(k * 100 + log_n)
    results = [0, P - 1] + [int(v) for v in CD.draw(k, rng)]
    run_fib(ctx, oracle, k, log_n, blowup, ext, results[:k], seed=log_n)


def test_fib_bench_shape(ctx, oracle):
    """FibSmall x 32, cubic, 2^22 rows, blowup 8: a 16 GiB LDE of random canonical words made on the device"""
    import torch
    k, log_n, blowup, ext = 32, 22, 8, 3
    live0 = ctx.mem_stats()[0]
    n, N, ce = 1 << log_n, (1 << log_n) * blowup, 2 << log_n
    g = torch.Generator(device="cuda").manual_seed(22)
    dev = torch.randint(-2**63, 2**63 - 1, (N * 2 * k,), dtype=torch.int64, device="cuda", generator=g)
    dev[(dev < 0) & (dev >= -(2**32 - 1))] = 5   # words of p or more (signed -(2^32 - 1) .. -1) -> canonical
    rng = np.random.default_rng(22)
    results = [0, P - 1] + [int(v) for v in CD.draw(k - 2, rng)]
    coeffs = CD.draw((5 * k, ext), rng)
    m = ctx.mat_wrap_device(dev.data_ptr(), N, 2 * k)
    fo = ctx.eval_constraints_fib(k, results, log_n, blowup, ext, m, coeffs)
    go = eval_generic(ctx, CD.fib_desc(k, n, results), log_n, blowup, ext, m, None, coeffs, None, True)
    rows = sample_rows(ce, rng, count=256)
    got, gen = fo.read_rows(rows), go.read_rows(rows)
    ls = rows.astype(np.int64) << 2
    cur, nxt = m.read_rows(ls.astype(np.uint64)), m.read_rows(((ls + blowup) % N).astype(np.uint64))
    want = oracle.eval_constraint_rows(CD.fib_desc(k, n, results), n, blowup, ext, coeffs, None, rows, cur, nxt)
    assert np.array_equal(got, want)
    assert np.array_equal(gen, want)
    for o in (fo, go, m):
        o.free()
    del dev
    torch.cuda.empty_cache()
    assert ctx.mem_stats()[0] == live0


@pytest.mark.parametrize("k", [2, 32])
def test_fib_accumulator_edges(ctx, oracle, k):
    """aimed T, B0 and B1 accumulators (combine_model.fib_aims): aimed CE rows 4 apart, so that the next-state LDE row of one
    is never the current row of another; ext 1, the coefficients of the aimed accumulator fib_mult, the others random"""
    log_n, blowup, ext = 9, 8, 1
    n, ce, N = 1 << log_n, 2 << log_n, (1 << log_n) * blowup
    aims = M.fib_aims(k, random.Random(k))
    rng = np.random.default_rng(k)
    results = [0, P - 1] + [int(v) for v in CD.draw(k - 2, rng)]
    for acc in ("T", "B0", "B1"):
        rows = [row for a, _, row in aims if a == acc]
        assert 4 * len(rows) <= ce
        lde = CD.draw((N, 2 * k), rng)
        coeffs = CD.draw((5 * k, ext), rng)
        if acc == "T":
            mult = M.fib_mult(2 * k)
            coeffs[: 2 * k, 0] = mult                                 # tc0_j, tc1_j interleaved as the kernel reads them
        elif acc == "B0":
            coeffs[2 * k: 4 * k, 0] = M.fib_mult(2 * k)               # b0a_j, b0b_j (columns 2j, 2j+1 at step 0)
        else:
            coeffs[4 * k:, 0] = M.fib_mult(k)                         # b1_j (column 2j+1 at step n-1)
        for r, vals in enumerate(rows):
            ls, lx = (4 * r) << 2, ((4 * r) << 2) + blowup
            v = np.array(vals, dtype=np.uint64)
            if acc == "T":   # t0 = nxt.x - cur.x - cur.y, t1 = nxt.y - cur.y - nxt.x: cur = 0, nxt.x = t0, nxt.y = t1 + t0
                lde[ls] = 0
                lde[lx, 0::2] = v[0::2]
                lde[lx, 1::2] = [(int(a) + int(b)) % P for a, b in zip(v[1::2], v[0::2])]
            elif acc == "B0":
                lde[ls] = v
            else:
                lde[ls, 1::2] = v
        run_fib(ctx, oracle, k, log_n, blowup, ext, results, seed=k, lde=lde, coeffs=coeffs, windows_too=False)


# ---- generic descriptions, one per evaluator path ----
@pytest.mark.parametrize("groups", [1, 3, 4, 5, 8, 9])
def test_boundary_groups(ctx, oracle, groups):
    for log_n, blowup, ext in ((4, 8, 1), (7, 4, 3), (10, 2, 2)):
        rng = np.random.default_rng(groups * 10 + log_n)
        run_generic(ctx, oracle, CD.boundary_groups(1 << log_n, groups, rng), log_n, blowup, ext, seed=groups + log_n)


@pytest.mark.parametrize("groups", [1, 3, 4, 5, 8, 9])
def test_aux_boundary_groups(ctx, oracle, groups):
    for log_n, blowup, ext in ((4, 4, 1), (6, 8, 2), (9, 4, 3)):
        rng = np.random.default_rng(groups * 10 + log_n)
        run_generic(ctx, oracle, CD.aux_groups(1 << log_n, groups, rng), log_n, blowup, ext, seed=groups + log_n)


@pytest.mark.parametrize("count", [1, 2, 8])
def test_exemptions(ctx, oracle, count):
    for log_n, blowup, ext in ((4, 4, 3), (8, 8, 1)):
        run_generic(ctx, oracle, CD.exemptions(1 << log_n, count, np.random.default_rng(count)), log_n, blowup, ext, seed=count)


def test_periodic_columns(ctx, oracle):
    for log_n, blowup, ext in ((3, 4, 2), (6, 8, 3), (11, 4, 1)):
        run_generic(ctx, oracle, CD.periodic(1 << log_n, np.random.default_rng(log_n)), log_n, blowup, ext, seed=log_n)


@pytest.mark.parametrize("ceb", [2, 4, 8, 16, 32, 64, 128])
def test_ce_blowup(ctx, oracle, ceb):
    log_n = 4 if ceb >= 64 else 6
    ext = (1, 2, 3)[ceb.bit_length() % 3]
    desc = CD.ce_blowup(1 << log_n, ceb, np.random.default_rng(ceb))
    for blowup in (ceb, 2 * ceb) if ceb < 128 else (ceb,):    # LDE shift 0, then 1
        run_generic(ctx, oracle, desc, log_n, blowup, ext, seed=ceb + blowup)


@pytest.mark.parametrize("name", CD.PROGRAMS)
def test_programs(ctx, oracle, name):
    run_generic(ctx, oracle, CD.program(name, 64, np.random.default_rng(1)), 6, 4, 2, seed=3)


def test_register_limits(ctx, oracle):
    run_generic(ctx, oracle, CD.main_registers(32, np.random.default_rng(1)), 5, 4, 3, seed=1)
    run_generic(ctx, oracle, CD.aux_registers(32, np.random.default_rng(2)), 5, 4, 3, seed=2)


@pytest.mark.parametrize("ext", [1, 2, 3])
def test_aux_segment_large(ctx, oracle, ext):
    """2^17 CE rows: compared on sampled rows"""
    run_generic(ctx, oracle, CD.aux_groups(1 << 16, 9, np.random.default_rng(ext)), 16, 2, ext, seed=ext, with_windows=False)


# ---- refusals ----
def test_refusals(ctx):
    n, log_n, blowup = 64, 6, 4
    live0 = ctx.mem_stats()[0]
    desc = CD.boundary_groups(n, 3, np.random.default_rng(0))
    A = TV.Air(desc)
    ncc = len(A.degrees) + len(A.asserts)
    cf = np.zeros((ncc, 2), dtype=np.uint64)
    ce = n * 2
    lde = np.zeros((n * blowup, A.w), dtype=np.uint64)
    full = ctx.mat_from_host_columns(lde.T)
    win = ctx.mat_from_host_columns(window_lde(lde, 0, 64, 1, blowup).T)
    narrow = ctx.mat_from_host_columns(window_lde(lde, 0, 64, 1, blowup)[:, :-1].T)
    for row0, cr, m in ((0, 0, full), (ce - 32, 64, win), (ce, 64, win), (0, 32, win), (0, 64, full), (0, 64, narrow)):
        with pytest.raises(wf.WfError):
            ctx.eval_constraints_window(desc, log_n, blowup, 2, m, None, cf, None, row0, cr)
        assert ctx.mem_stats()[0] == live0 + 3
    fl = np.zeros((n * blowup, 4), dtype=np.uint64)
    ffull = ctx.mat_from_host_columns(fl.T)
    fwin = ctx.mat_from_host_columns(window_lde(fl, 0, 64, 1, blowup).T)
    fc = np.zeros((10, 2), dtype=np.uint64)
    for k, row0, cr, m in ((0, 0, 0, ffull), (2, 0, 0, fwin), (2, 0, 32, fwin), (2, ce - 32, 64, fwin), (2, 64, 0, ffull),
                           (3, 0, 0, ffull), (2, 0, 64, ffull)):
        with pytest.raises(wf.WfError):
            ctx.eval_constraints_fib(k, [1, 2, 3], log_n, blowup, 2, m, fc, row0, cr)
        assert ctx.mem_stats()[0] == live0 + 5
    ok = ctx.eval_constraints_fib(2, [1, 2], log_n, blowup, 2, fwin, fc, 0, 64)
    assert ok.rows == 64
    for m in (full, win, narrow, ffull, fwin, ok):
        m.free()
    assert ctx.mem_stats()[0] == live0
