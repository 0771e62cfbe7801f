"""The oracle's constraint evaluation on chosen CE rows (wfo_eval_constraint_rows, the loop body of its prover) pinned to a
restatement in Python integers: the transition programs run through trace_validate_ref's interpreter; here only the
combination is restated: coefficients, e(x) / (x^n - 1), the group divisors x^a - b and the sequence values."""
import numpy as np
import pytest

import constraint_descs as CD
import trace_validate_ref as TV
from airs import P


def _interp(vals, O):
    """coefficients of the polynomial of degree < L through vals over the L-th roots of unity"""
    L = len(vals)
    w = O.root_of_unity(L.bit_length() - 1)
    inv_l, wi = pow(L, P - 2, P), pow(w, P - 2, P)
    return [inv_l * sum(int(v) * pow(wi, k * m, P) for k, v in enumerate(vals)) % P for m in range(L)]


def _horner(coeffs, x):
    y = 0
    for c in reversed(coeffs):
        y = (y * x + c) % P
    return y


def _emb(v, ext):
    return (int(v),) + (0,) * (ext - 1)


def last_outs(prog):
    """the program with only the last OUT of each constraint: the prover's OUT sets a constraint's value (result[dst] = r[a]),
    trace_validate_ref's run adds them"""
    seen, out = set(), []
    for ins in reversed(prog):
        if ins[0] == 4 and ins[1] in seen:
            continue
        seen |= {ins[1]} if ins[0] == 4 else set()
        out.append(ins)
    return out[::-1]


def ref_rows(O, desc, n, ext, coeffs, rand, rows, cur, nxt, acur=None, anxt=None):
    A = TV.Air(desc)
    A.prog, A.aux_prog = last_outs(A.prog), last_outs(A.aux_prog)
    ce = n << A.log_ce_blowup()
    w_ce, g = O.root_of_unity(ce.bit_length() - 1), O.root_of_unity(n.bit_length() - 1)
    cc = [tuple(int(v) for v in c) for c in np.asarray(coeffs).reshape(-1, ext)]
    k = len(rows)
    xs = [7 * pow(w_ce, int(i), P) % P for i in rows]
    obj = lambda a: np.asarray(a, dtype=np.uint64).astype(object)
    cur, nxt = obj(cur), obj(nxt)
    per = [np.array([_horner(_interp(col, O), pow(x, n // len(col), P)) for x in xs], dtype=object) for col in A.periodic]
    ac = an = []
    if A.aw:
        acur, anxt = obj(acur).reshape(k, A.aw, ext), obj(anxt).reshape(k, A.aw, ext)
        ac = [tuple(acur[:, c, q] for q in range(ext)) for c in range(A.aw)]
        an = [tuple(anxt[:, c, q] for q in range(ext)) for c in range(A.aw)]
    main, aux = TV.evaluate(A, [cur[:, c] for c in range(A.w)], [nxt[:, c] for c in range(A.w)], ac, an, per,
                            np.asarray(rand).reshape(-1, ext) if A.aw else None, ext, k)
    n_mt, n_tr = len(A.degrees), len(A.degrees) + len(A.aux_degrees)
    order = lambda asserts: sorted(range(len(asserts)), key=lambda i: (asserts[i][2], asserts[i][1], asserts[i][0]))
    out = []
    for r, x in enumerate(xs):
        t = (0,) * ext
        for j, v in enumerate(main):
            t = TV.e_add(t, TV.e_mul(cc[j], _emb(v[r], ext)))
        for j, v in enumerate(aux):
            t = TV.e_add(t, TV.e_mul(tuple(c[r] for c in v), cc[n_mt + j]))
        ex = 1
        for s in range(n - A.exemptions, n):
            ex = ex * (x - pow(g, s, P)) % P
        acc = TV.e_mul(t, _emb(pow(pow(x, n, P) - 1, P - 2, P) * ex % P, ext))
        base = n_tr
        for seg, asserts in ((0, A.asserts), (1, A.aux_asserts)):
            for idx, i in enumerate(order(asserts)):
                col, first, stride, vals = asserts[i]
                vals = [v[:ext] if seg else _emb(v[0], ext) for v in vals]
                a = 1 if stride == 0 else n // stride
                if len(vals) == 1:
                    val = vals[0]
                else:   # the interpolant of the values over the size-a subgroup at x g^-first
                    y = x * pow(g, (P - 2) * first, P) % P
                    val = tuple(_horner(_interp([v[q] for v in vals], O), y) for q in range(ext))
                frame = _emb(cur[r, col], ext) if seg == 0 else tuple(int(acur[r, col, q]) for q in range(ext))
                div = (pow(x, a, P) - (pow(g, a * first, P) if first else 1)) % P
                term = TV.e_mul(TV.e_sub(frame, val), cc[base + idx])
                acc = TV.e_add(acc, TV.e_mul(term, _emb(pow(div, P - 2, P), ext)))
            base += len(asserts)
        out.append([int(v) for v in acc])
    return np.array(out, dtype=np.uint64)


def frames(A, n, blowup, ext, rows, rng):
    """random frames with edge words for CE rows `rows` (the evaluator reads whatever LDE rows it is given)"""
    k = len(rows)
    cur, nxt = CD.draw((k, A.w), rng), CD.draw((k, A.w), rng)
    acur = anxt = None
    if A.aw:
        acur, anxt = CD.draw((k, A.aw * ext), rng), CD.draw((k, A.aw * ext), rng)
    return cur, nxt, acur, anxt


def cases(n, rng):
    yield "fib_small_x3", CD.fib_desc(3, n, [0, P - 1, 5])
    for gr in (1, 4, 9):
        yield f"boundary_groups_{gr}", CD.boundary_groups(n, gr, rng)
        yield f"aux_groups_{gr}", CD.aux_groups(n, gr, rng)
    yield "exemptions_8", CD.exemptions(n, 8, rng)
    yield "ce_blowup_8", CD.ce_blowup(n, 8, rng)
    yield "periodic", CD.periodic(n, rng)
    for name in CD.PROGRAMS:
        yield name, CD.program(name, n, rng)
    yield "main_registers", CD.main_registers(n, rng)
    yield "aux_registers", CD.aux_registers(n, rng)


@pytest.mark.parametrize("n", [16, 32, 64])
@pytest.mark.parametrize("ext", [1, 2, 3])
def test_oracle_rows_equal_the_python_restatement(oracle, n, ext):
    rng = np.random.default_rng(n * 10 + ext)
    for name, desc in cases(n, rng):
        A = TV.Air(desc)
        ceb = 1 << A.log_ce_blowup()
        ce, blowup = n * ceb, max(8, ceb)
        rows = np.unique(np.concatenate([[0, ce // 2 - 1, ce // 2, ce - 1], rng.integers(0, ce, 12)])).astype(np.uint64)
        ncc = len(A.degrees) + len(A.aux_degrees) + len(A.asserts) + len(A.aux_asserts)
        coeffs = CD.draw((ncc, ext), rng)
        rand = CD.draw((max(A.nr, 1), ext), rng)
        rand[0] = P - 1
        cur, nxt, acur, anxt = frames(A, n, blowup, ext, rows, rng)
        got = oracle.eval_constraint_rows(desc, n, blowup, ext, coeffs, rand, rows, cur, nxt, acur, anxt)
        want = ref_rows(oracle, desc, n, ext, coeffs, rand, rows, cur, nxt, acur, anxt)
        assert np.array_equal(got, want), name


def test_oracle_rows_refuse_bad_shapes(oracle):
    desc = CD.ce_blowup(16, 8, np.random.default_rng(0))
    z = np.zeros((1, CD.MAIN_W), dtype=np.uint64)
    c = np.zeros((20, 1), dtype=np.uint64)
    with pytest.raises(ValueError):   # blowup below ce_blowup
        oracle.eval_constraint_rows(desc, 16, 4, 1, c, None, [0], z, z)
    with pytest.raises(ValueError):   # a row outside the CE domain
        oracle.eval_constraint_rows(desc, 16, 8, 1, c, None, [16 * 8], z, z)
