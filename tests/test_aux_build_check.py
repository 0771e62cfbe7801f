"""Aux build descriptions without a GPU: wf_aux_build_check accepts perm_rap's build and names the reason for each class of
rejection; fuzzed descriptions only ever get WF_OK / WF_ERR_INVALID back; the CPU reference of the build semantics
(tests/aux_build_ref.cpp) reproduces perm_rap's Python builder; the scan kernels keep their state in registers."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import airs  # noqa: E402
import aux_builds as ab  # noqa: E402
import winterfell_b200 as wf  # noqa: E402

WF_OK, WF_ERR_INVALID = 0, -2
P = wf.P


def _perm_rap_like(build_fn):
    """perm_rap's AIR with a build whose columns build_fn(B) writes (B: AuxBuild of the AIR's shape)."""
    desc = airs.perm_rap(64)[0]
    B = ab.AuxBuild(3, airs.PERM_RAP_AUX_WIDTH, 1, 2)
    build_fn(B)
    return desc, B.build()


def _sums(B, first=None):
    """three running-sum columns with numerator 1; `first` writes column 0's program instead"""
    for j in range(3):
        c = B.column(ab.RUNNING_SUM)
        if j == 0 and first:
            first(c)
        else:
            c.num(c.const(1))


def test_perm_rap_build_passes_and_rejections_are_named():
    desc, bd = airs.perm_rap(64)[0], ab.perm_rap_build()
    assert wf.aux_build_check(desc, bd, 6) == (WF_OK, "")

    def reason(d, b, log_n=6):
        rc, msg = wf.aux_build_check(d, b, log_n)
        assert rc == WF_ERR_INVALID and msg, (rc, msg)
        return msg

    assert reason(desc, bd[:-1]) == "malformed aux build description"                       # structure: truncated
    assert reason(desc, np.concatenate([bd, [0]]).astype(np.uint64)) == "malformed aux build description"   # trailing word
    b = bd.copy(); b[0] = 2
    assert reason(desc, b) == "aux build width does not match the AIR's aux width"
    assert reason(airs.mulfib2(64)[0], bd) == "single-segment AIR: it has no aux segment to build"
    b = bd.copy(); b[2] = P                                                                 # the constant pool's only word
    assert reason(desc, b) == "aux build constant is not a canonical field element"
    b = bd.copy(); b[3] = 3                                                                 # column 0's kind
    assert reason(desc, b) == "unknown aux column kind"
    b = bd.copy(); b[4] = P                                                                 # column 0's init0
    assert reason(desc, b) == "aux column init is not a canonical field element"
    b = bd.copy(); b[7] = 97                                                                # column 0's num_regs > AUX_MAX_REGS
    assert reason(desc, b) == "aux build register count out of range"
    assert reason(desc, bd, 1) == "bad arguments"
    # register ranges: the column's own aux register, a later column's, a register past num_regs, an unwritten temporary
    unwritten = lambda c: (setattr(c, "next_reg", c.next_reg + 1), c.num(c.next_reg - 1))  # noqa: E731
    for bad in (lambda c: c.num(c.acur(0)), lambda c: c.num(c.anxt(2)), lambda c: c.num(c.next_reg + 5), unwritten):
        assert "reads a register out of range, an aux column >= its own" in reason(*_perm_rap_like(lambda B: _sums(B, bad)))
    d, b = _perm_rap_like(lambda B: _sums(B, lambda c: c.prog.append((airs.ADD, 0, 0, 0)) or c.num(0)))
    assert reason(d, b) == "aux build program writes a register outside its temporaries"
    d, b = _perm_rap_like(lambda B: _sums(B, lambda c: c.den(c.const(2))))
    assert reason(d, b) == "aux build column needs exactly one numerator (OUT 0)"
    d, b = _perm_rap_like(lambda B: _sums(B, lambda c: (c.num(c.const(2)), c.num(c.const(3)))))
    assert reason(d, b) == "aux build column needs exactly one numerator (OUT 0)"
    d, b = _perm_rap_like(lambda B: _sums(B, lambda c: (c.num(c.const(2)), c.den(c.const(3)), c.den(c.const(4)))))
    assert reason(d, b) == "aux build column has more than one denominator (OUT 1)"
    d, b = _perm_rap_like(lambda B: _sums(B, lambda c: c.prog.append((airs.OUT, 2, c.const(1), 0))))
    assert reason(d, b) == "aux build OUT selects neither numerator (0) nor denominator (1)"
    d, b = _perm_rap_like(lambda B: _sums(B, lambda c: c.prog.append((5, c.next_reg, 0, 0))))
    assert reason(d, b) == "unknown aux build opcode"
    # reads of earlier columns at rows i and i + 1 are allowed
    d, b = _perm_rap_like(lambda B: [B.column(ab.POINTWISE).num(0)] + [
        (lambda c: c.num(c.mul(c.acur(0), c.anxt(0 if j == 1 else 1))))(B.column(ab.RUNNING_PRODUCT)) for j in (1, 2)])
    assert wf.aux_build_check(d, b, 6) == (WF_OK, "")


@pytest.mark.parametrize("seed", range(4))
def test_fuzzed_build_descriptions_never_crash(seed):
    rng = np.random.default_rng(2000 + seed)
    interesting = np.array([0, 1, 2, 3, 4, 5, 7, 8, 95, 96, 97, 255, 1 << 20, (1 << 32) - 1, 1 << 63, P - 1, P, (1 << 64) - 1], dtype=np.uint64)
    desc = airs.perm_rap(64)[0]
    bases = [ab.perm_rap_build(),
             _perm_rap_like(lambda B: [B.column(ab.POINTWISE).num(0)] + [
                 (lambda c: c.den(c.sub(c.mul(c.acur(0), c.anxt(0)), c.rnd(1))) or c.num(c.per(0)))(B.column(ab.RUNNING_SUM, (1, 2, 3)))
                 for _ in (1, 2)])[1]]
    seen = {WF_OK: 0, WF_ERR_INVALID: 0}
    for d in bases:
        for _ in range(600):
            m = d.copy()
            kind = rng.integers(0, 5)
            if kind == 0:
                m = m[: rng.integers(0, len(m))]
            elif kind == 1:
                m = np.concatenate([m, rng.choice(interesting, size=rng.integers(1, 9))])
            elif kind == 2:
                for i in rng.integers(0, len(m), size=rng.integers(1, 4)):
                    m[i] = rng.choice(interesting)
            elif kind == 3:
                for i in rng.integers(0, len(m), size=rng.integers(1, 4)):
                    m[i] = np.uint64((int(m[i]) + int(rng.integers(-2, 3))) % (1 << 64))
            else:
                for i in rng.integers(0, len(m), size=rng.integers(1, 6)):
                    m[i] = np.uint64(int(rng.integers(0, 1 << 63)) * 2 + int(rng.integers(0, 2)))
            rc, msg = wf.aux_build_check(desc, np.ascontiguousarray(m, dtype=np.uint64), int(rng.integers(3, 12)))
            assert rc in (WF_OK, WF_ERR_INVALID), (rc, msg)
            assert (rc == WF_OK) == (msg == "")
            seen[rc] += 1
    assert seen[WF_ERR_INVALID] > 500 and seen[WF_OK] > 0


@pytest.mark.parametrize("d", [1, 2, 3])
def test_reference_aux_build_matches_perm_rap_builder(oracle, d):
    desc, trace, builder = airs.perm_rap(64)
    rand = oracle.rand_elems((2, d), 40 + d)
    got = ab.reference(desc, ab.perm_rap_build(), trace, rand)
    assert np.array_equal(got, builder.reference(rand))
    assert np.array_equal(got, builder(rand))


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "winterfell_b200", "_build", "auxbuild.o")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not (os.path.exists(OBJ) and os.path.exists(CUOBJDUMP)), reason="objects not built or no cuobjdump")
def test_scan_kernels_keep_state_in_registers():
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
    scans = {n: ops for n, ops in fns.items() if "aux_scan_" in n}
    assert len(scans) == 3 * 3 * 2, list(fns)          # reduce / carry / apply x D in {1,2,3} x {product, sum}
    for name, ops in scans.items():
        assert not any(o.startswith(("LDL", "STL")) for o in ops), name
        assert any(o.startswith("SHFL") for o in ops), name    # warp-level scan through shuffles
