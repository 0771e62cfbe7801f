"""LINEAR_RECURRENCE aux columns (a[i+1] = m_i * a[i] + t_i) without a GPU: the CPU reference of the build semantics
(tests/linrec_build_ref.cpp) against a Python-integer restatement, the checks of wf_aux_build_check and their messages, a fuzz
run over descriptions with kind-4 columns, and the affine scan kernels keep their state in registers."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import airs  # noqa: E402
import linrec_builds as ab  # noqa: E402
import linrec_airs as la  # noqa: E402
import winterfell_b200 as wf  # noqa: E402

WF_OK, WF_ERR_INVALID = 0, -2
P = wf.P


# ---- the extension fields of f64 as Python integers: x^2 = x - 2 (quadratic), x^3 = x + 1 (cubic) ----
def e_add(a, b): return tuple((x + y) % P for x, y in zip(a, b))


def e_mul(a, b):
    d = len(a)
    c = [0] * (2 * d - 1)
    for i in range(d):
        for j in range(d):
            c[i + j] += a[i] * b[j]
    for k in range(2 * d - 2, d - 1, -1):   # reduce x^k
        if d == 2:
            c[k - 1] += c[k]
            c[k - 2] -= 2 * c[k]
        else:
            c[k - 2] += c[k]
            c[k - 3] += c[k]
    return tuple(v % P for v in c[:d])


def e_inv(a):
    if not any(a):
        return a
    r, e, base = (1,) + (0,) * (len(a) - 1), P ** len(a) - 2, a
    while e:
        if e & 1:
            r = e_mul(r, base)
        base = e_mul(base, base)
        e >>= 1
    return r


def restated(cols, n, d, rand, tr):
    """linrec-shaped columns (kind, init, m(i, regs), num(i, regs), den(i, regs) or None) over E as Python integers"""
    out = []
    for kind, init, m_of, num_of, den_of in cols:
        a, col = tuple(init[:d]), []
        for i in range(n):
            col.append(a)
            regs = {"tr": tr, "rand": rand, "prev": out, "i": i, "nx": (i + 1) % n}
            t = num_of(regs)
            if den_of is not None:
                t = e_mul(t, e_inv(den_of(regs)))
            a = e_mul(a, t) if kind == ab.RUNNING_PRODUCT else e_add(e_mul(m_of(regs), a), t)
        out.append(col)
    return np.array(out, dtype=np.uint64)


def test_python_extension_arithmetic_is_the_oracles(oracle):
    for d in (2, 3):
        a, b = oracle.rand_elems((2, d), 90 + d)
        assert e_mul(tuple(int(v) for v in a), tuple(int(v) for v in b)) == tuple(int(v) for v in oracle.ext_mul(a, b))
        assert e_inv(tuple(int(v) for v in a)) == tuple(int(v) for v in oracle.ext_inv(a))


@pytest.mark.parametrize("d", [1, 2, 3])
def test_reference_keeps_the_running_kinds(oracle, d):
    # for kinds 0-2 the reference with kind 4 gives the columns of the existing one (tests/aux_build_ref.cpp)
    import aux_builds
    desc, trace, _ = airs.perm_rap(64)
    rand = oracle.rand_elems((2, d), 60 + d)
    assert np.array_equal(ab.reference(desc, ab.perm_rap_build(), trace, rand),
                          aux_builds.reference(desc, aux_builds.perm_rap_build(), trace, rand))
    ldesc, ltr, lbuild, _ = la.linrec(64)
    with pytest.raises(ValueError):   # and the existing one still does not take kind 4
        aux_builds.reference(ldesc, lbuild, ltr, rand)


def _emb(v, d): return (int(v) % P,) + (0,) * (d - 1)


@pytest.mark.parametrize("d", [1, 2, 3])
def test_reference_matches_python_restatement(oracle, d):
    n = 64
    desc, tr, build, builder = la.linrec(n, seed=3 + d)
    rand = oracle.rand_elems((2, d), 50 + d)
    R = [tuple(int(v) for v in r) for r in rand]
    xa = lambda g: e_add(_emb(g["tr"][2, g["i"]], d), R[0])   # noqa: E731
    got = ab.reference(desc, build, tr, rand)
    assert np.array_equal(got, builder(rand))
    want = restated([
        (ab.RUNNING_PRODUCT, (1, 0, 0), None, xa, None),
        (ab.LINEAR_RECURRENCE, (0, 0, 0), xa, lambda g: g["prev"][0][g["i"]], None),
        (ab.LINEAR_RECURRENCE, (0, 0, 0), lambda g: R[1], lambda g: _emb(g["tr"][0, g["i"]], d), None),
        (ab.LINEAR_RECURRENCE, (0, 0, 0), lambda g: _emb(1 - int(g["tr"][1, g["i"]]), d), lambda g: _emb(g["tr"][0, g["i"]], d), None),
    ], n, d, R, tr)
    assert np.array_equal(got, want)
    # m = 0 resets: R restarts with v after every row whose selector is 1
    i = int(np.flatnonzero(tr[1, :-1])[0])
    assert tuple(got[3, i + 1]) == _emb(tr[0, i], d)
    # a second shape: a denominator with zeros, m = p - 1, reads of column 0 at rows i and i + 1 (the wrap row too), an init
    # non-zero in every word
    B = ab.AuxBuild(3, 2, 0, 2)
    init = [int(v) for v in oracle.rand_elems((d,), 7)] + [0] * (3 - d)
    c0 = B.column(ab.LINEAR_RECURRENCE, init)
    c0.multiplier(c0.cur(1))
    c0.num(c0.cur(0))
    c0.den(c0.add(c0.cur(2), c0.rnd(0)))
    c1 = B.column(ab.LINEAR_RECURRENCE, init)
    c1.multiplier(c1.const(P - 1))
    c1.num(c1.add(c1.mul(c1.acur(0), c1.anxt(0)), c1.rnd(1)))
    A = airs.AirBuilder(3)
    A.constraint(A.sub(A.nxt(0), A.cur(0)), 1)
    A.assert_single(0, 0, 0)
    X = A.aux(2, 2)
    X.constraint(X.sub(X.anxt(0), X.acur(0)), 1)
    X.assert_single(0, 0, (0, 0, 0))
    desc2, build2 = A.build(), B.build()
    rand2 = rand.copy()
    rand2[0, 1:] = 0
    tr2 = oracle.rand_elems((3, n), 8)
    tr2[1, [0, 9, n - 2]] = 0
    tr2[2, [3, n // 2]] = (P - int(rand2[0, 0])) % P
    R2 = [tuple(int(v) for v in r) for r in rand2]
    want2 = restated([
        (ab.LINEAR_RECURRENCE, init, lambda g: _emb(g["tr"][1, g["i"]], d), lambda g: _emb(g["tr"][0, g["i"]], d),
         lambda g: e_add(_emb(g["tr"][2, g["i"]], d), R2[0])),
        (ab.LINEAR_RECURRENCE, init, lambda g: _emb(P - 1, d),
         lambda g: e_add(e_mul(g["prev"][0][g["i"]], g["prev"][0][g["nx"]]), R2[1]), None),
    ], n, d, R2, tr2)
    got2 = ab.reference(desc2, build2, tr2, rand2)
    assert np.array_equal(got2, want2)
    # m = 0 at row 0: a[1] = t_0 whatever init is; a zero denominator at row 3: t_3 = 0, a[4] = m_3 a[3]
    assert tuple(got2[0, 1]) == e_mul(_emb(tr2[0, 0], d), e_inv(e_add(_emb(tr2[2, 0], d), R2[0])))
    assert tuple(got2[0, 4]) == e_mul(_emb(tr2[1, 3], d), tuple(int(v) for v in got2[0, 3]))


def _linrec_with(col_fn, kind=ab.LINEAR_RECURRENCE):
    """the example AIR's description with a build whose column 1 col_fn(c) writes (columns 0, 2, 3 as in linrec)"""
    desc = la.linrec(64)[0]
    B = ab.AuxBuild(3, la.LINREC_AUX_WIDTH, 0, la.LINREC_NUM_RANDS)
    d = B.column(ab.RUNNING_PRODUCT, (1, 0, 0))
    d.num(d.add(d.cur(2), d.rnd(0)))
    col_fn(B.column(kind))
    for _ in (2, 3):
        c = B.column(ab.LINEAR_RECURRENCE)
        c.multiplier(c.rnd(1))
        c.num(c.cur(0))
    return desc, B.build()


def _reason(desc, build, log_n=6):
    rc, msg = wf.aux_build_check(desc, build, log_n)
    assert rc == WF_ERR_INVALID and msg, (rc, msg)
    return msg


def test_linrec_build_passes_and_new_rejections_are_named():
    desc, build = la.linrec(64)[:3:2]
    assert wf.aux_build_check(desc, build, 6) == (WF_OK, "")
    assert _reason(*_linrec_with(lambda c: c.num(c.cur(0)))) == "aux build LINEAR_RECURRENCE column has no multiplier (OUT 2)"
    assert _reason(*_linrec_with(lambda c: (c.multiplier(c.rnd(1)), c.num(c.cur(0)), c.multiplier(c.cur(1))))) == \
        "aux build LINEAR_RECURRENCE column has more than one multiplier (OUT 2)"
    assert _reason(*_linrec_with(lambda c: (c.multiplier(c.rnd(1)), c.num(c.cur(0)), c.prog.append((airs.OUT, 3, c.cur(0), 0))))) == \
        "aux build OUT selects neither numerator (0), denominator (1) nor multiplier (2)"
    # the rules every kind keeps: one numerator, at most one denominator, registers readable
    assert _reason(*_linrec_with(lambda c: c.multiplier(c.rnd(1)))) == "aux build column needs exactly one numerator (OUT 0)"
    assert _reason(*_linrec_with(lambda c: (c.multiplier(c.rnd(1)), c.num(c.cur(0)), c.den(c.cur(1)), c.den(c.cur(2))))) == \
        "aux build column has more than one denominator (OUT 1)"
    assert "reads a register out of range, an aux column >= its own" in _reason(
        *_linrec_with(lambda c: (c.multiplier(c.acur(1)), c.num(c.cur(0)))))
    # a denominator and reads of the column before it at rows i and i + 1 are allowed
    ok = _linrec_with(lambda c: (c.multiplier(c.anxt(0)), c.num(c.acur(0)), c.den(c.cur(2))))
    assert wf.aux_build_check(*ok, 6) == (WF_OK, "")


def test_other_kinds_keep_their_verdicts():
    desc, build = la.linrec(64)[:3:2]
    col1 = 3 + 6 + 8   # [aw, nC, one constant], column 0: [kind, init x3, num_regs, nI], two instructions
    assert build[col1] == ab.LINEAR_RECURRENCE
    for k in (3, 7, 5, 1 << 63):
        b = build.copy()
        b[col1] = k
        assert _reason(desc, b) == "unknown aux column kind"
    # OUT 2 in a running or pointwise column keeps the message it had before kind 4 existed
    for kind in (ab.POINTWISE, ab.RUNNING_PRODUCT, ab.RUNNING_SUM):
        msg = _reason(*_linrec_with(lambda c: (c.num(c.cur(0)), c.multiplier(c.rnd(1))), kind))
        assert msg == "aux build OUT selects neither numerator (0) nor denominator (1)"
    # a kind-4 column turned into a running sum: its OUT 2 is now out of place
    b = build.copy()
    b[col1] = ab.RUNNING_SUM
    assert _reason(desc, b) == "aux build OUT selects neither numerator (0) nor denominator (1)"


@pytest.mark.parametrize("seed", range(3))
def test_fuzzed_linrec_descriptions_never_crash(seed):
    rng = np.random.default_rng(4000 + seed)
    interesting = np.array([0, 1, 2, 3, 4, 5, 7, 8, 95, 96, 97, 255, 1 << 20, (1 << 32) - 1, 1 << 63, P - 1, P, (1 << 64) - 1], dtype=np.uint64)
    desc, build = la.linrec(64)[:3:2]
    bases = [build, _linrec_with(lambda c: (c.multiplier(c.anxt(0)), c.num(c.acur(0)), c.den(c.cur(2))))[1]]
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
    assert any("multiplier" in r for r in reasons), reasons


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "winterfell_b200", "_build", "auxbuild.o")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not (os.path.exists(OBJ) and os.path.exists(CUOBJDUMP)), reason="objects not built or no cuobjdump")
def test_affine_scan_kernels_keep_state_in_registers():
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
    scans = {n: ops for n, ops in fns.items() if "aux_affine_" in n}
    assert len(scans) == 3 * 3, list(fns)                 # reduce / carry / apply x D in {1,2,3}
    for name, ops in scans.items():
        assert not any(o.startswith(("LDL", "STL")) for o in ops), name
        assert any(o.startswith("SHFL") for o in ops), name    # warp-level scan through shuffles
    assert len([n for n in fns if "aux_scan_" in n]) == 3 * 3 * 2   # the running kinds keep their own kernels
