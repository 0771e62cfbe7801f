"""Hand-written AIR descriptions for the row-by-row tests of the constraint evaluators (test_oracle_constraint_rows.py,
test_gpu_constraint_rows.py), each named for the evaluator path it reaches, and the words their LDEs and coefficients are
drawn from. The evaluators do not check that an LDE satisfies its AIR, so any words serve as frames."""
import numpy as np

from airs import P, AirBuilder

# words at the edges of the field's encodings: 0, 1, p - 1, 2^32 - 1, 2^32, p - 2^32
EDGE_WORDS = (0, 1, P - 1, 2**32 - 1, 2**32, P - 2**32)


def draw(shape, rng, edge_share=0.5):
    """canonical words: each an edge word with probability edge_share, else uniform in [0, p)"""
    a = rng.integers(0, P, size=shape, dtype=np.uint64)
    pick = rng.random(shape) < edge_share
    a[pick] = np.array(EDGE_WORDS, dtype=np.uint64)[rng.integers(0, len(EDGE_WORDS), size=int(pick.sum()))]
    return a


def fib_desc(k, n, results):
    """the description of FibSmall x k (tests/airs.py fib_small_x) with any public results; its program reuses two
    temporaries per pair, as the oracle's fib_air does, so that k = 32 stays within the 160 registers"""
    A = AirBuilder(2 * k)
    A.pub = [int(r) for r in results]
    w, t = 2 * k, 4 * k
    for j in range(k):
        A.prog += [(0, t, 2 * j, 2 * j + 1), (1, t + 1, w + 2 * j, t), (4, 2 * j, t + 1, 0),
                   (0, t, 2 * j + 1, w + 2 * j), (1, t + 1, w + 2 * j + 1, t), (4, 2 * j + 1, t + 1, 0)]
        A.degrees += [(1, []), (1, [])]
        A.assert_single(2 * j, 0, j + 1)
        A.assert_single(2 * j + 1, 0, j + 1)
        A.assert_single(2 * j + 1, n - 1, results[j])
    A.next_reg = t + 2
    return A.build()


# ---- one main program (12 columns) shared by the boundary-group, exemption and ce_blowup descriptions ----
MAIN_W = 12


def _main(degree=1):
    A = AirBuilder(MAIN_W)
    A.constraint(A.sub(A.nxt(0), A.add(A.cur(0), A.cur(1))), degree)
    A.constraint(A.sub(A.nxt(1), A.mul(A.cur(1), A.cur(2))), 2 if degree < 2 else degree)
    A.constraint(A.add(A.mul(A.cur(11), A.nxt(11)), A.cur(5)), 2)
    return A


def _group_keys(n):
    """nine boundary groups (BTreeMap key (stride, first_step)): (key, columns) with columns of their own, so that no two
    assertions cover one cell; group 0 and 3 have several entries, 4 and 6 are sequences whose row shift wraps"""
    return [((0, 0), (0, 1, 2)), ((0, n - 1), (3,)), ((0, n // 2 + 1), (4,)), ((4, 1), (5, 6)), ((n // 4, 3), (7,)),
            ((8, 3), (8,)), ((n // 2, 1), (9,)), ((0, 1), (10,)), ((n, 5), (11,))]


def boundary_groups(n, groups, rng):
    """`groups` main boundary groups of single, periodic and sequence assertions (n >= 16)"""
    A = _main()
    for (stride, first), cols in _group_keys(n)[:groups]:
        for c in cols:
            if stride == 0:
                A.assert_single(c, first, int(draw(1, rng)[0]))
            elif stride in (n // 4, n // 2):
                A.assert_sequence(c, first, stride, [int(v) for v in draw(n // stride, rng)])
            else:
                A.assert_periodic(c, first, stride, int(draw(1, rng)[0]))
    return A.build()


def exemptions(n, count, rng):
    A = _main()
    A.exemptions = count
    A.assert_single(0, 0, int(draw(1, rng)[0]))
    return A.build()


def ce_blowup(n, ceb, rng):
    """constraint 0 declared of degree ceb: a constraint-evaluation blowup of ceb (>= 2)"""
    A = _main(ceb)
    A.assert_single(3, n - 1, int(draw(1, rng)[0]))
    A.assert_sequence(7, 2, n // 4, [int(v) for v in draw(4, rng)])
    return A.build()


def periodic(n, rng):
    """periodic columns of lengths 2, 4, n/2 and n; the second constraint's cycles raise ce_blowup to 4"""
    A = AirBuilder(3)
    A.periodic = [[int(v) for v in draw(L, rng)] for L in (2, 4, n // 2, n)]
    A.constraint(A.sub(A.nxt(0), A.add(A.mul(A.cur(0), A.per(0)), A.per(3))), 1, [n])
    A.constraint(A.sub(A.mul(A.nxt(1), A.per(1)), A.mul(A.cur(2), A.per(2))), 1, [2, n // 2, 4])
    A.constraint(A.mul(A.cur(2), A.per(1)), 1, [4])
    A.assert_single(0, 0, 3)
    A.assert_periodic(2, 1, 4, int(draw(1, rng)[0]))
    return A.build()


def program(name, n, rng):
    """transition programs at the edges of the instruction set"""
    A = AirBuilder(4)
    if name == "empty":                       # a declared constraint and no instruction: it evaluates to 0
        A.degrees.append((1, []))
    elif name == "out_of_input":              # OUT straight from frame registers
        A.prog.append((4, 0, A.cur(2), 0))
        A.prog.append((4, 1, A.nxt(3), 0))
        A.degrees += [(1, []), (1, [])]
    elif name == "several_outs":              # constraint 0 is the sum of three OUTs
        t = A.mul(A.cur(0), A.nxt(1))
        A.prog += [(4, 0, t, 0), (4, 0, A.cur(3), 0), (4, 1, A.nxt(0), 0), (4, 0, A.sub(A.cur(1), A.nxt(2)), 0)]
        A.degrees += [(2, []), (1, [])]
    elif name == "no_out":                    # constraint 1 has no OUT
        A.prog.append((4, 0, A.add(A.cur(0), A.nxt(3)), 0))
        A.degrees += [(1, []), (1, [])]
    elif name == "constants":                 # constants 0 and p - 1
        z, m = A.const(0), A.const(P - 1)
        A.constraint(A.add(A.mul(A.cur(0), m), A.nxt(0)), 1)
        A.constraint(A.sub(A.mul(z, A.cur(1)), A.mul(m, A.cur(2))), 1)
        A.constraint(A.mul(m, m), 1)
    A.assert_single(1, 0, int(draw(1, rng)[0]))
    return A.build()


PROGRAMS = ("empty", "out_of_input", "several_outs", "no_out", "constants")


def main_registers(n, rng):
    """a main program that uses all 160 registers of the interpreter's register file"""
    A = AirBuilder(8)
    regs = list(range(16))
    while A.next_reg is None or A.next_reg < 160:
        a, b = regs[-1], regs[-2 - (len(regs) % 7)]
        regs.append((A.add, A.sub, A.mul)[len(regs) % 3](a, b))
    A.constraint(regs[-1], 2)
    A.constraint(regs[40], 1)
    A.assert_single(0, 0, int(draw(1, rng)[0]))
    assert A.next_reg == 160
    return A.build()


def _aux_main():
    A = AirBuilder(2)
    A.constraint(A.sub(A.nxt(0), A.add(A.cur(0), A.cur(1))), 1)
    return A


AUX_W = 12


def aux_groups(n, groups, rng, ext_words=3):
    """an aux segment of AUX_W columns and 2 random elements whose `groups` boundary groups cover the same keys as the main
    ones; the aux program mixes main and aux frame registers, a constant and both random elements"""
    A = _aux_main()
    A.assert_single(1, n - 1, int(draw(1, rng)[0]))
    X = A.aux(AUX_W, 2)
    g, a = X.rnd(0), X.rnd(1)
    X.constraint(X.sub(X.mul(X.anxt(0), X.add(X.cur(1), g)), X.mul(X.acur(0), X.add(X.nxt(0), a))), 2)
    X.constraint(X.sub(X.anxt(8), X.add(X.acur(4), X.mul(a, X.cur(0)))), 2)
    X.constraint(X.mul(X.acur(7), X.const(P - 1)), 1)
    for (stride, first), cols in _group_keys(n)[:groups]:
        for c in cols:
            if stride == 0:
                X.assert_single(c, first, tuple(int(v) for v in draw(3, rng)))
            elif stride in (n // 4, n // 2):
                X.assert_sequence(c, first, stride, [tuple(int(v) for v in draw(3, rng)) for _ in range(n // stride)])
            else:   # one value: a periodic assertion
                X.assert_sequence(c, first, stride, [tuple(int(v) for v in draw(3, rng))])
    return A.build()


def aux_registers(n, rng):
    """an aux program that uses all 96 registers of the interpreter's aux register file"""
    A = _aux_main()
    A.assert_single(0, 0, 1)
    X = A.aux(4, 2)
    regs = list(range(X.next_reg))
    while X.next_reg < 96:
        a, b = regs[-1], regs[-2 - (len(regs) % 5)]
        regs.append((X.add, X.sub, X.mul)[len(regs) % 3](a, b))
    X.constraint(regs[-1], 2)
    X.assert_single(2, 0, (1, 2, 3))
    assert X.next_reg == 96
    return A.build()
