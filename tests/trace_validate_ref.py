"""CPU restatement of the reference's debug-build trace checks, for the tests of wf_trace_validate:
Trace::validate (prover/src/trace/mod.rs:86-201) and ConstraintEvaluationTable::validate_transition_degrees
(prover/src/constraints/evaluation_table.rs:181-230, 421-477). It has its own description parser and its own program
evaluator (Python integers, every register a vector over all steps or CE rows); the transforms come from the oracle.
Returns the dictionary Context.trace_validate returns."""
import numpy as np

from airs import P

VALID, MAIN_ASSERTION, AUX_ASSERTION, MAIN_TRANSITION, AUX_TRANSITION, DEGREES, CE_DOMAIN = range(7)


class Air:
    def __init__(self, desc):
        d = [int(v) for v in desc]
        self.p = 0

        def rd():
            v = d[self.p]
            self.p += 1
            return v

        def degrees():
            out = []
            for _ in range(rd()):
                base, nc = rd(), rd()
                out.append((base, [rd() for _ in range(nc)]))
            return out

        def prog():
            return [tuple(rd() for _ in range(4)) for _ in range(rd())]

        def asserts(words):
            out = []
            for _ in range(rd()):
                col, first, stride, nv = rd(), rd(), rd(), rd()
                out.append((col, first, stride, [tuple(rd() for _ in range(words)) for _ in range(nv)]))
            return out

        self.w = rd()
        self.degrees = degrees()
        self.periodic = [[rd() for _ in range(rd())] for _ in range(rd())]
        self.consts = [rd() for _ in range(rd())]
        rd()  # number of registers
        self.prog = prog()
        self.asserts = asserts(1)
        self.pub = [rd() for _ in range(rd())]
        self.exemptions = rd()
        self.aw = self.nr = 0
        self.aux_degrees, self.aux_prog, self.aux_asserts = [], [], []
        if self.p < len(d):
            self.aw, self.nr = rd(), rd()
            self.aux_degrees = degrees()
            rd()
            self.aux_prog = prog()
            self.aux_asserts = asserts(3)

    def log_ce_blowup(self):
        r = 1
        for base, cyc in self.degrees + self.aux_degrees:
            bound = base + len(cyc) - 1
            r = max(r, (bound - 1).bit_length() if bound > 1 else 0)
        return r


# E = F[x] / (x^2 - x + 2) and F[x] / (x^3 - x - 1), as tuples of component vectors
def e_add(a, b): return tuple((x + y) % P for x, y in zip(a, b))
def e_sub(a, b): return tuple((x - y) % P for x, y in zip(a, b))


def e_mul(a, b):
    if len(a) == 1:
        return ((a[0] * b[0]) % P,)
    if len(a) == 2:
        return ((a[0] * b[0] - 2 * a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0] + a[1] * b[1]) % P)
    a0, a1, a2 = a
    b0, b1, b2 = b
    return ((a0 * b0 + a1 * b2 + a2 * b1) % P, (a0 * b1 + a1 * b0 + a1 * b2 + a2 * b1 + a2 * b2) % P, (a0 * b2 + a2 * b0 + a1 * b1 + a2 * b2) % P)


def run(prog, regs, consts, ncon, ext, m):
    """Runs a program over vectors of m values; returns each constraint's value (the sum of its OUTs)."""
    zero = np.zeros(m, dtype=object)
    out = [tuple(zero for _ in range(ext)) if ext else zero for _ in range(ncon)]
    for op, dst, a, b in prog:
        if op == 4:
            out[dst] = e_add(out[dst], regs[a]) if ext else (out[dst] + regs[a]) % P
        elif op == 3:
            c = np.full(m, consts[a], dtype=object)
            regs[dst] = tuple([c] + [zero] * (ext - 1)) if ext else c
        elif ext:
            regs[dst] = (e_add, e_sub, e_mul)[op](regs[a], regs[b])
        else:
            regs[dst] = ((regs[a] + regs[b]) % P, (regs[a] - regs[b]) % P, (regs[a] * regs[b]) % P)[op]
    return out


def evaluate(A, cur, nxt, acur, anxt, per, rand, ext, m):
    """Main (base field) and aux (E) constraint values over m rows of frames. cur / nxt: [w] vectors, acur / anxt: [aw][ext]."""
    regs = dict(enumerate(list(cur) + list(nxt) + list(per)))
    main = run(A.prog, regs, A.consts, len(A.degrees), 0, m)
    aux = []
    if A.aw:
        zero = np.zeros(m, dtype=object)
        emb = lambda v: tuple([v] + [zero] * (ext - 1))
        rv = [tuple(np.full(m, int(rand[j][q]), dtype=object) for q in range(ext)) for j in range(A.nr)]
        ar = [emb(v) for v in list(cur) + list(nxt)] + list(acur) + list(anxt) + [emb(v) for v in per] + rv
        aux = run(A.aux_prog, dict(enumerate(ar)), A.consts, len(A.aux_degrees), ext, m)
    return main, aux


def _cells(a, n):
    col, first, stride, vals = a
    for k in range(n // stride if stride else 1):
        yield k, first + k * stride, vals[0 if len(vals) == 1 else k]


def check_trace(desc, trace, aux=None, rand=None, ext=1):
    A = Air(desc)
    n = trace.shape[1]
    T = np.asarray(trace, dtype=np.uint64).astype(object)
    n_tr = len(A.degrees) + len(A.aux_degrees)
    rep = {"kind": VALID, "index": 0, "step": 0, "column": 0, "first_failing_step": [None] * n_tr, "msg": ""}
    X = np.asarray(aux, dtype=np.uint64).astype(object) if A.aw else None
    steps = n - A.exemptions
    idx = np.arange(steps)
    cur, nxt = [T[c, :steps] for c in range(A.w)], [T[c, 1:steps + 1] for c in range(A.w)]
    per = [np.array(col, dtype=object)[idx % len(col)] for col in A.periodic]
    acur = [tuple(X[c, :steps, q] for q in range(ext)) for c in range(A.aw)]
    anxt = [tuple(X[c, 1:steps + 1, q] for q in range(ext)) for c in range(A.aw)]
    main, auxv = evaluate(A, cur, nxt, acur, anxt, per, rand, ext, steps)
    vals = [v != 0 for v in main] + [np.logical_or.reduce([c != 0 for c in v]) for v in auxv]
    for j, bad in enumerate(vals):
        nz = np.flatnonzero(bad)
        rep["first_failing_step"][j] = int(nz[0]) if nz.size else None
    for seg, asserts in ((0, A.asserts), (1, A.aux_asserts if A.aw else [])):
        for i, a in enumerate(asserts):
            for k, step, v in _cells(a, n):
                got = (int(T[a[0], step]),) if seg == 0 else tuple(int(X[a[0], step, q]) for q in range(ext))
                if got != tuple(v[:len(got)]):
                    vs = str(v[0]) if seg == 0 or ext == 1 else "(" + ", ".join(str(x) for x in v[:ext]) + ")"
                    rep.update(kind=AUX_ASSERTION if seg else MAIN_ASSERTION, index=i, step=step, column=a[0],
                               msg=f"trace does not satisfy assertion {'aux_trace' if seg else 'main_trace'}({a[0]}, {step}) == {vs}")
                    return rep
    fails = [(s, j) for j, s in enumerate(rep["first_failing_step"]) if s is not None]
    if fails:
        s, j = min(fails)
        nm = len(A.degrees)
        rep.update(kind=MAIN_TRANSITION if j < nm else AUX_TRANSITION, index=j if j < nm else j - nm, step=s,
                   msg=f"{'main' if j < nm else 'auxiliary'} transition constraint {j if j < nm else j - nm} did not evaluate to ZERO at step {s}")
    return rep


def check_degrees(desc, trace, aux=None, rand=None, ext=1):
    """(expected, actual, kind, msg) of validate_transition_degrees; kind VALID when both checks pass."""
    from oracle import oracle as O
    A = Air(desc)
    n = trace.shape[1]
    log_n = n.bit_length() - 1
    ceb = 1 << A.log_ce_blowup()
    ce = n * ceb
    lde = O.lde_rows(O.interpolate_columns(np.asarray(trace, dtype=np.uint64)), ceb).T.astype(object)   # [w, ce]
    rows = np.arange(ce)
    nx = (rows + ceb) % ce
    cur, nxt = [lde[c] for c in range(A.w)], [lde[c, nx] for c in range(A.w)]
    acur = anxt = []
    if A.aw:
        X = np.asarray(aux, dtype=np.uint64).reshape(A.aw, n * ext)
        alde = O.lde_rows(O.interpolate_columns(X, ext), ceb, ext).T.astype(object)   # [aw * ext, ce]
        acur = [tuple(alde[c * ext + q] for q in range(ext)) for c in range(A.aw)]
        anxt = [tuple(alde[c * ext + q, nx] for q in range(ext)) for c in range(A.aw)]
    w_ce = O.root_of_unity((ce).bit_length() - 1)
    xs = [7 * pow(w_ce, i, P) % P for i in range(ce)]
    per = []
    for col in A.periodic:   # the periodic polynomial (interpolated over the L-th roots of unity) at x^(n/L)
        L = len(col)
        coeffs = [int(v) for v in O.interpolate_poly(np.array(col, dtype=np.uint64))]
        ys = []
        for x in xs:
            y, xn = 0, pow(x, n // L, P)
            for cf in reversed(coeffs):
                y = (y * xn + cf) % P
            ys.append(y)
        per.append(np.array(ys, dtype=object))
    main, auxv = evaluate(A, cur, nxt, acur, anxt, per, rand, ext, ce)
    g = O.root_of_unity(log_n)
    f = []
    for x in xs:   # 1 / divisor = prod_k (x - g^(n-k)) / (x^n - 1)
        num = 1
        for k in range(1, A.exemptions + 1):
            num = num * (x - pow(g, n - k, P)) % P
        f.append(num * pow((pow(x, n, P) - 1) % P, P - 2, P) % P)
    f = np.array(f, dtype=object)

    def degree(v):
        c = O.interpolate_poly(np.array([int(t) for t in (v * f) % P], dtype=np.uint64))
        nz = np.flatnonzero(c)
        return int(nz[-1]) if nz.size else 0

    actual = [degree(v) for v in main] + [max(degree(c) for c in v) for v in auxv]
    expected = []
    for base, cyc in A.degrees + (A.aux_degrees if A.aw else []):
        e = base * (n - 1) + sum((n // c) * (c - 1) for c in cyc)
        expected.append(e - (n - A.exemptions))
    if expected != actual:
        fmt = lambda v: "[" + ", ".join(f"{x:>3}" for x in v) + "]"
        return expected, actual, DEGREES, f"transition constraint degrees didn't match\nexpected: {fmt(expected)}\nactual:   {fmt(actual)}"
    dom = 1
    while dom < max(max(actual), n + 1):
        dom <<= 1
    if dom != ce:
        return expected, actual, CE_DOMAIN, f"incorrect constraint evaluation domain size; expected {dom}, but was {ce}"
    return expected, actual, VALID, ""


def validate(desc, trace, aux=None, rand=None, ext=1, check_degrees_too=True):
    """The full report of Context.trace_validate."""
    rep = check_trace(desc, trace, aux, rand, ext)
    rep["expected_degrees"] = rep["actual_degrees"] = None
    if check_degrees_too:
        e, a, kind, msg = check_degrees(desc, trace, aux, rand, ext)
        rep["expected_degrees"], rep["actual_degrees"] = e, a
        if rep["kind"] == VALID and kind != VALID:
            rep.update(kind=kind, index=0, step=0, column=0, msg=msg)
    return rep
