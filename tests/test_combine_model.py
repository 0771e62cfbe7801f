"""The accumulator, DEEP and fold model (combine_model.py) against plain integer arithmetic and the oracle, its aiming, and
the edge classes each kernel's generated inputs reach: every (kernel, class) cell is reached or listed with its reason."""
import random

import numpy as np
import pytest

import combine_model as M
import ntt_model as NM

P = M.P
DOT_K = (1, 2, 5, 64, 255)


def test_accumulator_equals_plain_sums(oracle):
    rng = random.Random(1)
    for k in DOT_K:
        rows = M.dot_rows(k, rng)
        rows += [("random", [rng.randrange(2**64) for _ in range(k)], [rng.randrange(2**64) for _ in range(k)])]
        for label, xs, ys in rows:
            w = M.dot(xs, ys)
            assert M.acc_value(w) == sum(x * y for x, y in zip(xs, ys)), (k, label)
            r = M.acc_reduce(w)
            assert r == sum(x * y for x, y in zip(xs, ys)) % P, (k, label)
            if all(x < P and y < P for x, y in zip(xs, ys)):
                want = 0
                for x, y in zip(xs, ys):
                    want = oracle.add(want, oracle.mul(x, y))
                assert r == want, (k, label)


@pytest.mark.parametrize("k", DOT_K)
def test_aimed_dot_products_reach_their_class(k):
    rng = random.Random(k)
    for label, xs, ys in M.dot_rows(k, rng):
        log = M.Log()
        M.acc_reduce(M.dot(xs, ys, log), k - 1, log)
        if label in M.REDUCE_CLASSES:
            assert ("dot", label) in log.hits, (k, label)
        elif label == "ripple":
            assert ("dot", "odd carry ripples through all-ones w1..w3") in log.hits or \
                ("dot", "even carry out of w3") in log.hits, k
        elif label == "all p - 1":
            assert ("dot", "w4 at kernel max") in log.hits


@pytest.mark.parametrize("d", [1, 2, 3])
def test_ood_and_deep_aims_reach_their_class(d):
    rng = random.Random(d)
    for label, z in M.structured_points(d):
        for comp in range(d):
            mult = M.ood_mults(z, comp)
            w4max = M.ood_max(mult) >> 128
            for cls, c in M.ood_thread_rows(mult, rng):
                log = M.Log()
                M.acc_reduce(M.dot(mult, c, log), w4max, log)
                assert all(v < P for v in c)
                if cls in M.REDUCE_CLASSES:
                    assert ("dot", cls) in log.hits, (label, comp, cls)
    for c in (2, 3, 8, 9, 64, 255):
        dc = M.deep_coeffs(c, d, d - 1)
        mult = [int(v) for v in dc[:, d - 1]]
        for cls, row in M.deep_rows(c, rng):
            log = M.Log()
            M.acc_reduce(M.dot(mult, row, log), M.deep_max(c) >> 128, log)
            assert all(v < P for v in row)
            if cls in M.REDUCE_CLASSES:
                assert ("dot", cls) in log.hits, (c, cls)


def test_extension_arithmetic_equals_oracle(oracle):
    rng = random.Random(3)
    for d in (2, 3):
        for _ in range(20):
            a, b = [rng.randrange(P) for _ in range(d)], [rng.randrange(P) for _ in range(d)]
            assert M.ext_mul(a, b) == [int(v) for v in oracle.ext_mul(np.array(a, dtype=np.uint64), np.array(b, dtype=np.uint64))]
            assert M.ext_inv(a) == [int(v) for v in oracle.ext_inv(np.array(a, dtype=np.uint64))]
            A, B = np.array([a, b], dtype=np.uint64), np.array([b, a], dtype=np.uint64)
            assert [[int(v) for v in r] for r in M.np_ext_mul(A, B)] == [M.ext_mul(a, b), M.ext_mul(b, a)]
        z = [rng.randrange(P) for _ in range(d)]
        cf = [rng.randrange(P) for _ in range(40)]
        assert M.horner(cf, z) == [int(v) for v in oracle.eval_poly_at(np.array(cf, dtype=np.uint64), np.array(z, dtype=np.uint64))]


@pytest.mark.parametrize("d", [1, 2, 3])
def test_vectorised_syn_div_equals_serial(oracle, d):
    for label, z in M.structured_points(d)[:3] + [("random", [random.Random(d).randrange(P) for _ in range(d)])]:
        s = oracle.rand_elems((37, d), 5 + d)
        b = np.array(z, dtype=np.uint64)
        assert np.array_equal(M.np_syn_div(s, b), M.host_syn_div(oracle, s, b, d)), label


@pytest.mark.parametrize("lognf", [1, 2, 3, 4])
def test_mini_dft_model_and_fold_aims(oracle, lognf):
    nf = 1 << lognf
    rng = random.Random(lognf)
    w = NM.root(lognf)
    for _ in range(4):
        x = [rng.randrange(P) for _ in range(nf)]
        F = [sum(x[k] * pow(w, j * k, P) for k in range(nf)) % P for j in range(nf)]
        out = M.mini_dft(x, lognf)
        assert [out[pos] for pos in range(nf)] == [F[NM.brev(pos, lognf)] for pos in range(nf)]
    # every aimed layer sees every butterfly class; the fold of the aimed layer equals the oracle's
    L, d = nf * 64, 2
    ev = M.fold_inputs(L, nf, d, np.random.default_rng(lognf))
    m = L // nf
    seen = {lvl: set() for lvl in range(lognf)}
    for i in range(m):
        for c in range(d):
            def obs(lvl, a, b, i=i):
                if lvl == i % lognf:
                    seen[lvl] |= NM.classify_pairs(np.array(a, dtype=np.uint64), np.array(b, dtype=np.uint64))
            M.mini_dft([int(ev[i + k * m, c]) for k in range(nf)], lognf, obs)
    for lvl in range(lognf):
        assert seen[lvl] == set(NM.PAIR_CLASSES), (lvl, set(NM.PAIR_CLASSES) - seen[lvl])


KERNELS = ("wf_acc_ops_dev", "ood_partial", "deep_sum", "fib_constraints")
UNREACHED = {
    ("ood_partial", "odd carry ripples through all-ones w1..w3"):
        "the multipliers are the fixed powers z^r and the aim fixes the final sum only; bits 32..127 of an intermediate "
        "sum all ones before a term is a 2^-96 event per term",
    ("deep_sum", "odd carry ripples through all-ones w1..w3"):
        "the aimed rows fix the final sum through (p-1, p-1) terms followed by two solving terms; no intermediate sum has "
        "bits 32..127 all ones (wf_acc_ops_dev covers the ripple with aimed prefixes)",
    ("deep_sum", "m2 = 1"):
        "the aimed multipliers are p - 1 and 1, whose low halves are 0 and 1: x0 y1 + x1 y0 < 2^64 "
        "(wf_acc_ops_dev covers it)",
}
UNREACHED[("fib_constraints", "odd carry ripples through all-ones w1..w3")] = UNREACHED[("deep_sum", "odd carry ripples through all-ones w1..w3")]
UNREACHED[("fib_constraints", "m2 = 1")] = UNREACHED[("deep_sum", "m2 = 1")]
FIB_K = (2, 3, 32)   # the widths test_gpu_constraint_rows.py aims the FibSmall kernel at


def kernel_log():
    log = M.Log()
    rng = random.Random(11)
    for k in DOT_K:
        for _, xs, ys in M.dot_rows(k, rng):
            M.acc_reduce(M.dot(xs, ys, log, "wf_acc_ops_dev"), k - 1, log, "wf_acc_ops_dev")
    for d in (1, 2, 3):
        for _, z in M.structured_points(d):
            for comp in range(d):
                mult = M.ood_mults(z, comp)
                for _, c in M.ood_thread_rows(mult, rng):
                    M.acc_reduce(M.dot(mult, c, log, "ood_partial"), M.ood_max(mult) >> 128, log, "ood_partial")
    for c in (2, 9, 64, 255):
        mult = [P - 1] * (c - 1) + [1]
        for _, row in M.deep_rows(c, rng):
            M.acc_reduce(M.dot(mult, row, log, "deep_sum"), M.deep_max(c) >> 128, log, "deep_sum")
    for k in FIB_K:
        for acc, _, row in M.fib_aims(k, random.Random(k)):
            mult = M.fib_mult(len(row))
            M.acc_reduce(M.dot(mult, row, log, "fib_constraints"), M.deep_max(len(row)) >> 128, log, "fib_constraints")
    return log


@pytest.mark.parametrize("k", FIB_K)
def test_fib_aims_reach_their_class(k):
    K0 = M.fib_k0(k)
    for acc, cls, row in M.fib_aims(k, random.Random(k)):
        log = M.Log()
        r = M.acc_reduce(M.dot(M.fib_mult(len(row)), row, log), M.deep_max(len(row)) >> 128, log)
        assert all(0 <= v < P for v in row) and len(row) == (k if acc == "B1" else 2 * k)
        if cls in M.REDUCE_CLASSES:
            assert ("dot", cls) in log.hits, (k, acc, cls)
        elif cls == "reduce(a0) = K0":
            assert r == K0
        elif cls == "reduce(a0) < K0":
            assert r < K0


def test_coverage_matrix(capsys):
    log = kernel_log()
    rows, missing = [], []
    for kern in KERNELS:
        for c in M.CLASSES:
            n = log.hits.get((kern, c), 0)
            if n:
                rows.append(f"{kern:16s} {c:44s} {n}")
            elif (kern, c) in UNREACHED:
                rows.append(f"{kern:16s} {c:44s} unreached: {UNREACHED[(kern, c)]}")
            else:
                missing.append((kern, c))
    with capsys.disabled():
        print("\nAccumulator edge coverage (kernel, class, hits or why not):\n" + "\n".join(rows))
    assert not missing, missing
    # the export reaches every class, so a kernel's unreached cell is still covered on its own device functions
    assert all(log.hits.get(("wf_acc_ops_dev", c)) for c in M.CLASSES)
