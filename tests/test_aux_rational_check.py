"""RATIONAL_RECURRENCE aux columns (a[i+1] = (m_i a[i] + n_i) / (c_i a[i] + d_i)) without a GPU: the CPU reference of the build
semantics (tests/rational_build_ref.cpp) against a Python-integer restatement, zero denominators included, the checks of
wf_aux_build_check and their messages, a fuzz run over descriptions with kind-6 columns, and the Moebius scan kernels keep their
state in registers."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import airs  # noqa: E402
import linrec_airs as la  # noqa: E402
import rational_airs as ra  # noqa: E402
import rational_builds as rb  # noqa: E402
import winterfell_b200 as wf  # noqa: E402
from test_aux_linrec_check import e_add, e_inv, e_mul  # noqa: E402

WF_OK, WF_ERR_INVALID = 0, -2
P = wf.P


def _emb(v, d): return (int(v) % P,) + (0,) * (d - 1)


def restated_rational(init, n, d, m_of, n_of, c_of, d_of):
    """one RATIONAL_RECURRENCE column over E as Python integers, row after row, inv(0) = 0"""
    a, col = tuple(init[:d]), []
    for i in range(n):
        col.append(a)
        a = e_mul(e_add(e_mul(m_of(i), a), n_of(i)), e_inv(e_add(e_mul(c_of(i), a), d_of(i))))
    return col


@pytest.mark.parametrize("d", [1, 2, 3])
def test_reference_keeps_the_other_kinds(oracle, d):
    # for kinds 0-4 the reference gives the columns of tests/linrec_build_ref.cpp
    import linrec_builds
    rand = oracle.rand_elems((2, d), 60 + d)
    ldesc, ltr, lbuild, lbuilder = la.linrec(64)
    assert np.array_equal(rb.reference(ldesc, lbuild, ltr, rand), lbuilder(rand))
    desc, tr, build, _ = ra.rational(64)
    with pytest.raises(ValueError):   # and that one does not take kind 6
        linrec_builds.reference(desc, build, tr, rand)


@pytest.mark.parametrize("d", [1, 2, 3])
def test_reference_matches_python_restatement(oracle, d):
    n = 64
    desc, tr, build, builder = ra.rational(n, seed=3 + d, zeros=(7, 8, 40), zero_zero=(20,))
    rand = oracle.rand_elems((2, d), 50 + d)
    R = [tuple(int(v) for v in r) for r in rand]
    got = builder(rand)
    one = _emb(1, d)
    f = restated_rational((0, 0, 0), n, d, lambda i: R[0], lambda i: _emb(tr[0, i], d), lambda i: one, lambda i: R[1])
    g = restated_rational((1, 0, 0), n, d, lambda i: _emb(tr[1, i], d), lambda i: _emb(tr[0, i], d), lambda i: _emb(tr[2, i], d),
                          lambda i: _emb(tr[3, i], d))
    h, acc = [], (0,) * d
    for i in range(n):
        h.append(acc)
        acc = e_add(acc, e_mul(f[i], g[i]))
    assert np.array_equal(got, np.array([f, g, h], dtype=np.uint64))
    # the aimed rows reach their cases: G is 0 after a vanishing denominator (7, 8 consecutive, 40) and after the 0/0 row 20,
    # and non-zero elsewhere
    gz = {i + 1 for i in (7, 8, 20, 40)}
    assert all((got[1, i] == 0).all() == (i in gz) for i in range(n)), [i for i in range(n) if not got[1, i].any()]
    assert [int(v) for v in got[1, :, 0]] == ra.g_column(tr)


def test_reference_zero_map_denominator(oracle):
    # c = d = 0 at row 3 with a non-zero numerator: a[4] = 0, and the column goes on from there
    d, n = 2, 16
    B = rb.AuxBuild(3, 1, 0, 1)
    c = B.column(rb.RATIONAL_RECURRENCE, (5, 0, 0))
    c.multiplier(c.cur(0))
    c.num(c.cur(1))
    c.den_multiplier(c.cur(2))
    c.den(c.mul(c.cur(2), c.rnd(0)))
    A = airs.AirBuilder(3)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, 0)
    X = A.aux(1, 1)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (0, 0, 0))
    desc, build = A.build(), B.build()
    tr = oracle.rand_elems((3, n), 4)
    tr[2, 3] = 0                  # c = d = 0 at row 3
    rand = oracle.rand_elems((1, d), 9)
    R0 = tuple(int(v) for v in rand[0])
    got = rb.reference(desc, build, tr, rand)
    want = restated_rational((5, 0, 0), n, d, lambda i: _emb(tr[0, i], d), lambda i: _emb(tr[1, i], d), lambda i: _emb(tr[2, i], d),
                             lambda i: e_mul(_emb(tr[2, i], d), R0))
    assert np.array_equal(got, np.array([want], dtype=np.uint64))
    assert not got[0, 4].any() and got[0, 5].any()


def _rational_with(col_fn, kind=rb.RATIONAL_RECURRENCE):
    """the example AIR's description with a build whose column 1 col_fn(c) writes (columns 0 and 2 as in rational)"""
    desc = ra.rational(64)[0]
    B = rb.AuxBuild(5, ra.RATIONAL_AUX_WIDTH, 0, ra.RATIONAL_NUM_RANDS)
    f = B.column(rb.RATIONAL_RECURRENCE)
    f.multiplier(f.rnd(0))
    f.num(f.cur(0))
    f.den_multiplier(f.const(1))
    f.den(f.rnd(1))
    col_fn(B.column(kind))
    h = B.column(rb.RUNNING_SUM)
    h.num(h.mul(h.acur(0), h.acur(1)))
    return desc, B.build()


def _reason(desc, build, log_n=6):
    rc, msg = wf.aux_build_check(desc, build, log_n)
    assert rc == WF_ERR_INVALID and msg, (rc, msg)
    return msg


def _g(c, skip=()):
    if "m" not in skip:
        c.multiplier(c.cur(1))
    c.num(c.cur(0))
    if "c" not in skip:
        c.den_multiplier(c.cur(2))
    c.den(c.cur(3))


def test_rational_build_passes_and_new_rejections_are_named():
    desc, build = ra.rational(64)[:3:2]
    assert wf.aux_build_check(desc, build, 6) == (WF_OK, "")
    assert _reason(*_rational_with(lambda c: _g(c, "m"))) == "aux build RATIONAL_RECURRENCE column has no multiplier (OUT 2)"
    assert _reason(*_rational_with(lambda c: (_g(c), c.multiplier(c.cur(4))))) == \
        "aux build RATIONAL_RECURRENCE column has more than one multiplier (OUT 2)"
    assert _reason(*_rational_with(lambda c: _g(c, "c"))) == "aux build RATIONAL_RECURRENCE column has no denominator multiplier (OUT 3)"
    assert _reason(*_rational_with(lambda c: (_g(c), c.den_multiplier(c.acur(0))))) == \
        "aux build RATIONAL_RECURRENCE column has more than one denominator multiplier (OUT 3)"
    for k in (4, 5, 1 << 32):
        assert _reason(*_rational_with(lambda c: (_g(c), c.prog.append((airs.OUT, k, c.cur(0), 0))))) == \
            "aux build OUT selects neither numerator (0), denominator (1), multiplier (2) nor denominator multiplier (3)"
    # the rules every kind keeps: one numerator, at most one denominator, registers readable
    assert _reason(*_rational_with(lambda c: (c.multiplier(c.cur(1)), c.den_multiplier(c.cur(2))))) == \
        "aux build column needs exactly one numerator (OUT 0)"
    assert _reason(*_rational_with(lambda c: (_g(c), c.den(c.cur(2))))) == "aux build column has more than one denominator (OUT 1)"
    assert "reads a register out of range, an aux column >= its own" in _reason(
        *_rational_with(lambda c: (c.multiplier(c.acur(1)), c.num(c.cur(0)), c.den_multiplier(c.cur(2)))))
    # no denominator (d = 1), and reads of the column before it at rows i and i + 1 are allowed
    ok = _rational_with(lambda c: (c.multiplier(c.anxt(0)), c.num(c.acur(0)), c.den_multiplier(c.cur(2))))
    assert wf.aux_build_check(*ok, 6) == (WF_OK, "")


def test_other_kinds_keep_their_messages():
    desc, build = ra.rational(64)[:3:2]
    col1 = 3 + 6 + 20   # [aw, nC, one constant], column 0: [kind, init x3, num_regs, nI], five instructions
    assert build[col1] == rb.RATIONAL_RECURRENCE
    for k in (3, 5, 7, 1 << 63):
        b = build.copy()
        b[col1] = k
        assert _reason(desc, b) == "unknown aux column kind"
    # OUT 3 in a column of any other kind keeps the message it had before kind 6 existed
    for kind in (rb.POINTWISE, rb.RUNNING_PRODUCT, rb.RUNNING_SUM):
        assert _reason(*_rational_with(lambda c: (c.num(c.cur(0)), c.den_multiplier(c.cur(2))), kind)) == \
            "aux build OUT selects neither numerator (0) nor denominator (1)"
    assert _reason(*_rational_with(lambda c: (c.multiplier(c.cur(1)), c.num(c.cur(0)), c.den_multiplier(c.cur(2))),
                                   rb.LINEAR_RECURRENCE)) == "aux build OUT selects neither numerator (0), denominator (1) nor multiplier (2)"
    # the kind-6 column turned into a linear recurrence or a running sum: its OUT 3 (and OUT 2) are now out of place
    b = build.copy()
    b[col1] = rb.LINEAR_RECURRENCE
    assert _reason(desc, b) == "aux build OUT selects neither numerator (0), denominator (1) nor multiplier (2)"
    b[col1] = rb.RUNNING_SUM
    assert _reason(desc, b) == "aux build OUT selects neither numerator (0) nor denominator (1)"
    # a linear recurrence turned into a rational one lacks its OUT 3
    ldesc, lbuild = la.linrec(64)[:3:2]
    b = lbuild.copy()
    b[3 + 6 + 8] = rb.RATIONAL_RECURRENCE
    assert _reason(ldesc, b) == "aux build RATIONAL_RECURRENCE column has no denominator multiplier (OUT 3)"


@pytest.mark.parametrize("seed", range(3))
def test_fuzzed_rational_descriptions_never_crash(seed):
    rng = np.random.default_rng(6000 + seed)
    interesting = np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 95, 96, 97, 255, 1 << 20, (1 << 32) - 1, 1 << 63, P - 1, P, (1 << 64) - 1],
                           dtype=np.uint64)
    desc, build = ra.rational(64)[:3:2]
    bases = [build, _rational_with(lambda c: (c.multiplier(c.anxt(0)), c.num(c.acur(0)), c.den_multiplier(c.cur(2))))[1]]
    seen = {WF_OK: 0, WF_ERR_INVALID: 0}
    reasons = set()
    for d in bases:
        for _ in range(500):
            m = d.copy()
            mode = rng.integers(0, 5)
            if mode == 0:
                m = m[: rng.integers(0, len(m))]
            elif mode == 1:
                m = np.concatenate([m, rng.choice(interesting, size=rng.integers(1, 9))])
            elif mode == 2:
                for i in rng.integers(0, len(m), size=rng.integers(1, 4)):
                    m[i] = rng.choice(interesting)
            elif mode == 3:
                for i in rng.integers(0, len(m), size=rng.integers(1, 4)):
                    m[i] = np.uint64((int(m[i]) + int(rng.integers(-2, 3))) % (1 << 64))
            else:
                for i in rng.integers(0, len(m), size=rng.integers(1, 6)):
                    m[i] = np.uint64(int(rng.integers(0, 1 << 63)) * 2 + int(rng.integers(0, 2)))
            rc, msg = wf.aux_build_check(desc, np.ascontiguousarray(m, dtype=np.uint64), int(rng.integers(3, 12)))
            assert rc in (WF_OK, WF_ERR_INVALID), (rc, msg)
            assert (rc == WF_OK) == (msg == "")
            seen[rc] += 1
            reasons.add(msg)
    assert seen[WF_ERR_INVALID] > 400 and seen[WF_OK] > 0
    assert any("denominator multiplier" in r for r in reasons), reasons


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "winterfell_b200", "_build", "auxbuild.o")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not (os.path.exists(OBJ) and os.path.exists(CUOBJDUMP)), reason="objects not built or no cuobjdump")
def test_moebius_kernels_keep_state_in_registers():
    out = subprocess.run([CUOBJDUMP, "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fns[cur] = []
        elif cur and re.match(r"\s+/\*[0-9a-f]{4,6}\*/", line):
            fns[cur].append(re.sub(r"^\s+/\*[0-9a-f]+\*/\s+(@!?U?P[0-9T]\s+)?", "", line).split()[0])
    assert set(re.findall(r"arch = (sm_\w+)", out)) == {"sm_90a"}
    scans = {n: ops for n, ops in fns.items() if re.search(r"aux_moebius_(reduce|carry|apply)", n)}
    assert len(scans) == 3 * 3, list(fns)                 # reduce / carry / apply x D in {1,2,3}
    for name, ops in scans.items():
        assert not any(o.startswith(("LDL", "STL")) for o in ops), name
        assert any(o.startswith("SHFL") for o in ops), name    # warp-level scan through shuffles
    assert any(o.startswith("ATOMG") or o.startswith("RED") for o in fns[next(n for n in scans if "apply" in n)])
    assert len([n for n in fns if "aux_moebius_term_kernel" in n]) == 3
    # the other kinds keep their own kernels
    assert len([n for n in fns if "aux_scan_" in n]) == 3 * 3 * 2
    assert len([n for n in fns if "aux_affine_" in n]) == 3 * 3
    assert len([n for n in fns if "aux_term_kernel" in n]) == 3 * 2
