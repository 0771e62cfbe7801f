"""COUPLED_RECURRENCE groups (a[i+1] = M_i a[i] + t_i over k = 2..4 aux columns) without a GPU: the CPU reference of the build
semantics (tests/coupled_build_ref.cpp) against a Python-integer restatement for k = 2, 3, 4 and D = 1, 2, 3, the example AIR's
columns against its constraints, the checks of wf_aux_build_check and their messages (the other kinds' unchanged), a fuzz run
over descriptions with kinds 8 and 9, and the group scan kernels keep their state in registers."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import airs  # noqa: E402
import coupled_airs as ca  # noqa: E402
import coupled_builds as cb  # noqa: E402
import linrec_airs as la  # noqa: E402
import rational_airs as ra  # noqa: E402
import trace_validate_ref as R  # noqa: E402
import winterfell_b200 as wf  # noqa: E402
from test_aux_linrec_check import e_add, e_mul  # noqa: E402

WF_OK, WF_ERR_INVALID = 0, -2
P = wf.P
MSG_MEMBER = "aux build COUPLED_MEMBER column does not follow a COUPLED_RECURRENCE column or another member"
MSG_SIZE = "aux build COUPLED_RECURRENCE group has fewer than 2 or more than 4 columns"
MSG_MEMBER_PROG = "aux build COUPLED_MEMBER column has registers or instructions"
MSG_SLOT = "aux build COUPLED_RECURRENCE OUT selects a slot outside the group's t (0 .. k-1) and M (4 + 4r + c, r, c < k)"
MSG_REPEAT = "aux build COUPLED_RECURRENCE program writes an OUT slot more than once"


def _emb(v, d): return (int(v) % P,) + (0,) * (d - 1)


def trivial_air(w, aw, nr):
    """an AIR of w main and aw aux columns whose constraints any trace meets (the build is what is tested)"""
    A = airs.AirBuilder(w)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, 0)
    X = A.aux(aw, nr)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (1, 0, 0))
    return A.build()


def entry(k, r, c):
    """what M[r][c] of the generic group reads: mixes main columns, random elements, aux column 0 at rows i and i + 1, products,
    and unwritten (zero) slots"""
    return [("main", (r + c) % 4), ("rnd", r % 2), ("acur",), ("anxt",), ("mul", c % 4), None][(3 * r + 5 * c + k) % 6]


def t_entry(r): return [("main", 0), ("rnd", 0), ("main", 2), None][r]


def generic_group(k, inits, w=4, nr=2):
    """The build: column 0 POINTWISE P0 = x3 alpha, columns 1 .. k a group whose map is entry() / t_entry(), column k + 1 a
    RUNNING_SUM of the group's columns 0 and k - 1 at row i + 1 (a later column reads the group)."""
    Bd = cb.AuxBuild(w, k + 2, 0, nr)
    p0 = Bd.column(cb.POINTWISE)
    p0.num(p0.mul(p0.cur(3), p0.rnd(0)))
    g = Bd.group(k, inits)

    def reg(e):
        if e[0] == "main":
            return g.cur(e[1])
        if e[0] == "rnd":
            return g.rnd(e[1])
        if e[0] == "acur":
            return g.acur(0)
        if e[0] == "anxt":
            return g.anxt(0)
        return g.mul(g.cur(e[1]), g.rnd(1))
    for r in range(k):
        for c in range(k):
            if entry(k, r, c) is not None:
                g.m(r, c, reg(entry(k, r, c)))
        if t_entry(r) is not None:
            g.t(r, reg(t_entry(r)))
    h = Bd.column(cb.RUNNING_SUM)
    h.num(h.add(h.anxt(1), h.anxt(k)))
    return trivial_air(w, k + 2, nr), Bd.build()


def restated_generic(k, inits, tr, rand, d):
    """the columns of generic_group over E as Python integers, row after row"""
    n = tr.shape[1]
    R_ = [tuple(int(v) for v in r) for r in rand]
    p0 = [e_mul(_emb(tr[3, i], d), R_[0]) for i in range(n)]

    def val(e, i):
        if e is None:
            return (0,) * d
        if e[0] == "main":
            return _emb(tr[e[1], i], d)
        if e[0] == "rnd":
            return R_[e[1]]
        if e[0] == "acur":
            return p0[i]
        if e[0] == "anxt":
            return p0[(i + 1) % n]
        return e_mul(_emb(tr[e[1], i], d), R_[1])
    a = [tuple(int(v) % P for v in inits[r][:d]) for r in range(k)]
    cols = [[] for _ in range(k)]
    for i in range(n):
        for r in range(k):
            cols[r].append(a[r])
        nxt = []
        for r in range(k):
            y = val(t_entry(r), i)
            for c in range(k):
                y = e_add(y, e_mul(val(entry(k, r, c), i), a[c]))
            nxt.append(y)
        a = nxt
    h, acc = [], (0,) * d
    for i in range(n):
        h.append(acc)
        acc = e_add(acc, e_add(cols[0][(i + 1) % n], cols[k - 1][(i + 1) % n]))
    return np.array([p0] + cols + [h], dtype=np.uint64)


def _inits(k, seed):
    rng = np.random.default_rng(seed)
    return [tuple(int(v) for v in rng.integers(1, P, size=3, dtype=np.uint64)) for _ in range(k)]


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("k", [2, 3, 4])
def test_reference_matches_python_restatement(oracle, k, d):
    n = 48
    inits = [tuple(v if q < d else 0 for q, v in enumerate(i)) for i in _inits(k, 10 * k + d)]
    desc, build = generic_group(k, inits)
    assert wf.aux_build_check(desc, build, 6) == (WF_OK, "")
    tr = oracle.rand_elems((4, n), 100 * k + d)
    rand = oracle.rand_elems((2, d), 200 * k + d)
    got = cb.reference(desc, build, tr, rand)
    assert np.array_equal(got, restated_generic(k, inits, tr, rand, d))
    assert got[1:k + 1, 1:].any()
    assert got[1, :, d - 1].any()           # extension-valued for d > 1


@pytest.mark.parametrize("d", [1, 2, 3])
def test_reference_keeps_the_other_kinds(oracle, d):
    # for kinds 0-6 the reference gives the columns of tests/rational_build_ref.cpp, and that one does not take kind 8
    import rational_builds
    for desc, tr, build, _ in (ra.rational(64), la.linrec(64)):
        rand = oracle.rand_elems((2, d), 60 + d)
        assert np.array_equal(cb.reference(desc, build, tr, rand), rational_builds.reference(desc, build, tr, rand))
    desc, tr, build, _ = ca.coupled(64)
    with pytest.raises(ValueError):
        rational_builds.reference(desc, build, tr, oracle.rand_elems((3, d), 1))


@pytest.mark.parametrize("d", [1, 2, 3])
def test_example_air_columns_meet_its_constraints(oracle, d):
    n = 64
    desc, tr, build, builder = ca.coupled(n, seed=d)
    assert wf.aux_build_check(desc, build, 6) == (WF_OK, "")
    rand = oracle.rand_elems((ca.COUPLED_NUM_RANDS, d), 40 + d)
    aux = builder(rand)
    assert R.validate(desc, tr, aux, rand, d)["kind"] == R.VALID
    # (A, B) is the second-order recurrence u[i+2] = p_i u[i+1] + q_i u[i] + v_i with u[0] = 2, u[1] = 1
    u = [2, 1]
    for i in range(n):
        u.append((int(tr[1, i]) * u[-1] + int(tr[2, i]) * u[-2] + int(tr[0, i])) % P)
    assert [int(v) for v in aux[ca.A, :, 0]] == u[1:n + 1] and [int(v) for v in aux[ca.B, :, 0]] == u[:n]
    bad = aux.copy()
    bad[ca.Y1, 33, 0] = (int(bad[ca.Y1, 33, 0]) + 1) % P
    rep = R.validate(desc, tr, bad, rand, d)
    assert rep["kind"] == R.AUX_TRANSITION and rep["step"] in (32, 33), rep


def _with(fn):
    """a build over the example AIR's shape: column 0 POINTWISE, then whatever fn(B) appends, filled to the aux width with
    POINTWISE columns"""
    desc = ca.coupled(64)[0]
    Bd = cb.AuxBuild(5, ca.COUPLED_AUX_WIDTH, 0, ca.COUPLED_NUM_RANDS)
    c = Bd.column(cb.POINTWISE)
    c.num(c.cur(0))
    fn(Bd)
    while len(Bd.cols) < ca.COUPLED_AUX_WIDTH:
        c = Bd.column(cb.POINTWISE)
        c.num(c.cur(1))
    return desc, Bd.build()


def _reason(desc, build, log_n=6):
    rc, msg = wf.aux_build_check(desc, build, log_n)
    assert rc == WF_ERR_INVALID and msg, (rc, msg)
    return msg


def _full_group(B, k):
    g = B.group(k, [(1, 0, 0)] * k)
    for r in range(k):
        g.t(r, 0)
        for c in range(k):
            g.m(r, c, 0)
    return g


def _ok(desc, build):
    assert wf.aux_build_check(desc, build, 6) == (WF_OK, "")


def test_coupled_build_passes_and_new_rejections_are_named():
    desc, _, build, _ = ca.coupled(64)
    _ok(desc, build)
    z = [(1, 0, 0)] * 4
    for k in (2, 3, 4):   # every slot of a k-group, and an empty program (the zero map)
        _ok(*_with(lambda B: _full_group(B, k)))
        _ok(*_with(lambda B: B.group(k, z)))
    # a member after a column of another kind, or first
    assert _reason(*_with(lambda B: B.member())) == MSG_MEMBER
    Bd = cb.AuxBuild(5, ca.COUPLED_AUX_WIDTH, 0, ca.COUPLED_NUM_RANDS)
    Bd.member()
    Bd.group(2, z)
    for _ in range(4):
        Bd.column(cb.POINTWISE).num(0)
    assert _reason(desc, Bd.build()) == MSG_MEMBER
    # group sizes 1 and 5, also at the end of the description
    assert _reason(*_with(lambda B: B.group(1, z))) == MSG_SIZE
    assert _reason(*_with(lambda B: B.group(5, z * 2))) == MSG_SIZE
    Bd = cb.AuxBuild(5, ca.COUPLED_AUX_WIDTH, 0, ca.COUPLED_NUM_RANDS)
    for _ in range(6):
        Bd.column(cb.POINTWISE).num(0)
    Bd.group(1, z)
    assert _reason(desc, Bd.build()) == MSG_SIZE
    # a member with registers or instructions
    for regs, prog in ((1, []), (0, [(airs.OUT, 0, 0, 0)]), (30, [(airs.CONST, 29, 0, 0)])):
        def bad(B):
            B.group(2, z)
            B.cols[-1].next_reg, B.cols[-1].prog = regs, prog
        assert _reason(*_with(bad)) == MSG_MEMBER_PROG
    # OUT slots outside t and M of the group: t_r and M rows / columns >= k, and beyond M[3][3]
    for k, slot in ((2, 2), (2, 3), (2, 4 + 4 * 0 + 2), (2, 4 + 4 * 2 + 0), (3, 3), (3, 4 + 3), (3, 4 + 4 * 3 + 1), (4, 20),
                    (4, 1 << 32)):
        assert _reason(*_with(lambda B: B.group(k, z).prog.append((airs.OUT, slot, 0, 0)))) == MSG_SLOT, (k, slot)
    # a repeated slot, t or M
    for slot in (1, 4 + 4 + 1):
        assert _reason(*_with(lambda B: B.group(2, z).prog.extend([(airs.OUT, slot, 0, 0)] * 2))) == MSG_REPEAT
    # the rules every kind keeps: readable registers, and the columns < j rule (the leader reads no column of its group)
    g = lambda B: B.group(2, z)   # noqa: E731
    assert "reads a register out of range, an aux column >= its own" in _reason(
        *_with(lambda B: (lambda c: c.m(0, 0, c.acur(1)))(g(B))))
    assert "reads a register out of range, an aux column >= its own" in _reason(
        *_with(lambda B: (lambda c: c.t(1, c.anxt(2)))(g(B))))
    _ok(*_with(lambda B: (lambda c: (c.m(0, 0, c.acur(0)), c.t(1, c.anxt(0))))(g(B))))
    # a column after the group reads all of it
    def after(B):
        B.group(2, z)
        c = B.column(cb.RUNNING_SUM)
        c.num(c.mul(c.acur(1), c.anxt(2)))
    _ok(*_with(after))


def test_other_kinds_keep_their_messages():
    desc, _, build, _ = ca.coupled(64)
    starts, q = [], 2 + int(build[1])   # [aw, nC, constants], then per column [kind, init x3, num_regs, nI, program]
    for _ in range(int(build[0])):
        starts.append(q)
        q += 6 + 4 * int(build[q + 5])
    lead = starts[ca.A]
    assert build[lead] == cb.COUPLED_RECURRENCE and build[starts[ca.B]] == cb.COUPLED_MEMBER
    for k in (3, 5, 7, 10, 1 << 63):
        b = build.copy()
        b[lead] = k
        assert _reason(desc, b) == "unknown aux column kind"
    # OUT slots above 1 (above 2, above 3) in columns of kinds 0-6 keep the messages they had
    for kind, msg in ((cb.POINTWISE, "aux build OUT selects neither numerator (0) nor denominator (1)"),
                      (cb.RUNNING_PRODUCT, "aux build OUT selects neither numerator (0) nor denominator (1)"),
                      (cb.RUNNING_SUM, "aux build OUT selects neither numerator (0) nor denominator (1)"),
                      (cb.LINEAR_RECURRENCE, "aux build OUT selects neither numerator (0), denominator (1) nor multiplier (2)"),
                      (cb.RATIONAL_RECURRENCE,
                       "aux build OUT selects neither numerator (0), denominator (1), multiplier (2) nor denominator multiplier (3)")):
        for slot in (4, 9, 19):
            assert _reason(*_with(lambda B: (lambda c: (c.num(c.cur(0)), c.prog.append((airs.OUT, slot, 0, 0))))(B.column(kind)))) == msg
    # the leader turned into a linear recurrence: its OUT 4.. are out of place there; the one-column rules hold again
    b = build.copy()
    b[lead] = cb.LINEAR_RECURRENCE
    assert _reason(desc, b) == "aux build OUT selects neither numerator (0), denominator (1) nor multiplier (2)"
    # a linear recurrence column turned into a leader: a group of one
    ldesc, lbuild = la.linrec(64)[:3:2]
    b = lbuild.copy()
    b[3 + 6 + 8] = cb.COUPLED_RECURRENCE
    assert _reason(ldesc, b) == MSG_SIZE
    # the rational and linear examples still pass
    for desc2, _, build2, _ in (ra.rational(64), la.linrec(64)):
        _ok(desc2, build2)


@pytest.mark.parametrize("seed", range(3))
def test_fuzzed_coupled_descriptions_never_crash(seed):
    rng = np.random.default_rng(8000 + seed)
    interesting = np.array([0, 1, 2, 3, 4, 5, 7, 8, 9, 10, 19, 20, 23, 95, 96, 97, 255, 1 << 20, (1 << 32) - 1, 1 << 63, P - 1, P,
                            (1 << 64) - 1], dtype=np.uint64)
    desc, _, build, _ = ca.coupled(64)
    bases = [build, _with(lambda B: _full_group(B, 4))[1]]
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
    assert any("COUPLED" in r for r in reasons), reasons


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "winterfell_b200", "_build", "auxbuild.o")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not (os.path.exists(OBJ) and os.path.exists(CUOBJDUMP)), reason="objects not built or no cuobjdump")
def test_coupled_kernels_keep_state_in_registers():
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
    scans = {n: ops for n, ops in fns.items() if re.search(r"aux_coupled_(reduce|carry|apply)", n)}
    assert len(scans) == 3 * 3 * 3, list(fns)             # reduce / carry / apply x k in {2,3,4} x D in {1,2,3}
    for name, ops in scans.items():
        assert not any(o.startswith(("LDL", "STL")) for o in ops), name
        assert any(o.startswith("SHFL") for o in ops), name    # the map's rows and the state move between lanes by shuffles
    assert len([n for n in fns if "aux_coupled_term_kernel" in n]) == 3
    # the other kinds keep their own kernels
    assert len([n for n in fns if "aux_scan_" in n]) == 3 * 3 * 2
    assert len([n for n in fns if "aux_affine_" in n]) == 3 * 3
    assert len([n for n in fns if re.search(r"aux_moebius_(reduce|carry|apply)", n)]) == 3 * 3
    assert len([n for n in fns if "aux_moebius_term_kernel" in n]) == 3
    assert len([n for n in fns if "aux_term_kernel" in n]) == 3 * 2
