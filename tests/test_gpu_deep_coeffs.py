"""DEEP composition in coefficient form (wf_deep_compose_polys: combination of the coefficient matrices, synthetic division by
X - z and X - z*g as a device suffix scan, one LDE of the quotient; composer/mod.rs:67-210) against the evaluation form over the
LDEs of the same polynomials (wf_deep_compose): the two must agree bit for bit. The division is also checked against the
reference's serial syn_div (polynom/mod.rs:498-505) run on the host. The scan tile is 2048 rows: n = 8 and 2^11 are one tile,
2^12 and 2^13 two and four, 2^18 and 2^22 need the carry block to walk several tiles per thread. Trace lengths are powers of
two, so the tile count always is one as well."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import combine_model as M
import winterfell_b200 as wf

P = wf.P
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "winterfell_b200", "_build", "prover.o")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def _inputs(ctx, oracle, seed, ext, c, aw, kc, n):
    """Random coefficient matrices (main n x c, aux n x aw*ext, composition n x kc*ext), z and the DEEP coefficients."""
    main = ctx.mat_from_host_columns(oracle.rand_elems((c, n), seed))
    aux = ctx.mat_from_host_columns(oracle.rand_elems((aw, n * ext), seed + 1), ext_degree=ext) if aw else None
    cons = ctx.mat_from_host_columns(oracle.rand_elems((kc, n * ext), seed + 2), ext_degree=ext)
    z = oracle.rand_elems((ext,), seed + 3)
    coeffs = oracle.rand_elems((c + aw + kc, ext), seed + 4)
    return main, aux, cons, z, coeffs


@pytest.mark.gpu
@pytest.mark.parametrize("ext,c,aw,kc,log_n,log_b", [
    (1, 3, 0, 1, 3, 1),
    (2, 9, 1, 2, 3, 3),
    (3, 2, 2, 2, 3, 4),
    (3, 9, 0, 1, 10, 3),
    (2, 4, 0, 2, 10, 4),
    (1, 8, 1, 2, 12, 3),
    (3, 16, 1, 1, 12, 1),
    (3, 9, 0, 2, 18, 3),
    (2, 3, 1, 1, 18, 4),
    (1, 9, 0, 1, 22, 3),
    (3, 8, 1, 2, 22, 1),
])
def test_coefficient_form_matches_evaluation_form(ctx, oracle, ext, c, aw, kc, log_n, log_b):
    n = 1 << log_n
    main, aux, cons, z, coeffs = _inputs(ctx, oracle, 1000 * log_n + 10 * ext + aw, ext, c, aw, kc, n)
    zg = oracle.ext_mul(z, np.array([oracle.root_of_unity(log_n)] + [0] * (ext - 1), dtype=np.uint64)) if ext > 1 \
        else np.array([oracle.mul(int(z[0]), oracle.root_of_unity(log_n))], dtype=np.uint64)
    # OOD rows of the evaluation form: main columns at z / zg, then aux, then composition columns
    cur, nxt = [], []
    for m, col_ext in ((main, 1), (aux, ext), (cons, ext)):
        if m is not None:
            a, b = ctx.evaluate_at(m, ext, col_ext, z, zg)
            cur.append(a)
            nxt.append(b)
    ldes = [m.lde(log_b) if m is not None else None for m in (main, aux, cons)]
    want = ctx.deep_compose(ext, ldes[0], ldes[1], ldes[2], log_n, z, coeffs, np.concatenate(cur), np.concatenate(nxt))
    got = ctx.deep_compose_polys(ext, main, aux, cons, log_b, z, coeffs)
    assert got.rows == n << log_b and got.cols == ext
    assert np.array_equal(got.to_rows(), want.to_rows())
    for o in [main, aux, cons, want, got] + ldes:
        if o is not None:
            o.free()


@pytest.mark.gpu
@pytest.mark.parametrize("ext,log_n", [(1, 3), (3, 3), (2, 11), (3, 12), (1, 13)])
def test_division_matches_serial_syn_div(ctx, oracle, ext, log_n):
    n, c, aw, kc = 1 << log_n, 2, 1, 1
    main, aux, cons, z, coeffs = _inputs(ctx, oracle, 77 + log_n + ext, ext, c, aw, kc, n)
    deep = ctx.deep_compose_polys(ext, main, aux, cons, 1, z, coeffs)
    coef = deep.interpolate_with_offset(7).to_rows()   # the quotient's coefficients, 2n rows
    # S = sum_j coeffs_j p_j over the coefficients (component q of an extension column = base column j*ext + q)
    r = main.to_rows()
    cols = [r[:, j:j + 1] for j in range(c)]
    for m in (aux, cons):
        r = m.to_rows()
        cols += [r[:, j * ext:(j + 1) * ext] for j in range(r.shape[1] // ext)]
    s = np.zeros((n, ext), dtype=np.uint64)
    for j, col in enumerate(cols):
        for i in range(n):
            x = np.zeros(ext, dtype=np.uint64)
            x[:col.shape[1]] = col[i]
            t = oracle.ext_mul(coeffs[j], x) if ext > 1 else np.array([oracle.mul(int(coeffs[j][0]), int(x[0]))], dtype=np.uint64)
            s[i] = [(int(u) + int(v)) % P for u, v in zip(s[i], t)]
    zg = oracle.ext_mul(z, np.array([oracle.root_of_unity(log_n)] + [0] * (ext - 1), dtype=np.uint64)) if ext > 1 \
        else np.array([oracle.mul(int(z[0]), oracle.root_of_unity(log_n))], dtype=np.uint64)
    qz, qzg = M.host_syn_div(oracle, s, z, ext), M.host_syn_div(oracle, s, zg, ext)
    want = np.array([[(int(u) + int(v)) % P for u, v in zip(a, b)] for a, b in zip(qz, qzg)], dtype=np.uint64)
    assert np.array_equal(coef[:n], want)
    assert not coef[n:].any()
    for o in (main, aux, cons, deep):
        o.free()


@pytest.mark.skipif(not (os.path.exists(OBJ) and os.path.exists(CUOBJDUMP)), reason="objects not built or no cuobjdump")
def test_division_scan_kernels_keep_state_in_registers():
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
    scans = {n: ops for n, ops in fns.items() if "syn_div_" in n}
    assert len(scans) == 3 * 3, list(fns)   # reduce / carry / apply x D in {1, 2, 3}
    for name, ops in scans.items():
        assert not any(o.startswith(("LDL", "STL")) for o in ops), name
        assert any(o.startswith("SHFL") for o in ops), name   # warp-level scan through shuffles
