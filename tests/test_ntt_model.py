"""The transform-network model of tests/ntt_model.py (CPU): it computes what the oracle computes, bit for bit, and the
inputs it generates put the requested edge operands at the targeted steps, with every edge class reaching every step."""
import numpy as np
import pytest

import ntt_model as M


@pytest.mark.parametrize("log_n", list(range(1, 12)) + [12, 13, 17])
def test_model_equals_oracle_ntt(oracle, log_n):
    x = oracle.rand_elems((2, 1 << log_n), 40 + log_n)
    assert (M.Network(log_n).forward(x)[1] == oracle.evaluate_poly(x[1])).all()
    assert (M.Network(log_n, inverse=True).forward(x)[0] == oracle.interpolate_poly(x[0])).all()


@pytest.mark.parametrize("log_n,inverse", [(22, False), (22, True), (23, False), (24, True)])
def test_model_equals_oracle_large(oracle, log_n, inverse):
    # 2^22 = 11.11, 2^23 = 8 + 8.7, 2^24 = 8 + 8.8, one column
    net = M.Network(log_n, inverse)
    assert [p.log_s for p in net.passes] == {22: [11, 11], 23: [8, 8, 7], 24: [8, 8, 8]}[log_n]
    x = oracle.rand_elems((1, 1 << log_n), log_n)
    want = oracle.interpolate_poly(x[0]) if inverse else oracle.evaluate_poly(x[0])
    assert (net.forward(x)[0] == want).all()


@pytest.mark.parametrize("log_n,log_b", [(1, 1), (4, 3), (6, 2), (11, 3), (12, 1), (12, 3), (13, 2), (17, 1), (20, 2)])
def test_model_equals_oracle_lde(oracle, log_n, log_b):
    # three-pass LDEs are the three-pass transform with the pass-1 pre-scale and post twiddle of the two-pass LDE
    x = oracle.rand_elems((1, 1 << log_n), 7 * log_n + log_b)
    assert (M.Network(log_n, log_blowup=log_b).forward(x) == oracle.lde_rows(x, 1 << log_b).T).all()


def test_model_equals_oracle_interpolate_with_offset(oracle):
    for log_n in (3, 11, 12):
        x = oracle.rand_elems((1, 1 << log_n), log_n)
        assert (M.interpolate_with_offset(x, 7)[0] == oracle.interpolate_poly_with_offset(x[0], 7)).all()


def test_plans_follow_the_kernels():
    assert [M.radices(s) for s in range(1, 12)] == [[1], [2], [3], [3, 1], [3, 2], [3, 3], [3, 4], [4, 4], [3, 3, 3],
                                                    [3, 3, 4], [3, 4, 4]]
    assert [M.split_log(n) for n in (11, 12, 13, 17, 22)] == [(0, 11), (6, 6), (7, 6), (9, 8), (11, 11)]
    # mini_dft<4>'s shifts after its first layer are 2^(12 q), q = 1..7: gl_mul_2exp<36> and <60> among them
    p = M.Pass("p", 8, ((256,), (0,)), ((256,), (0,)))
    assert p._shift_k(0, 0)[:, 0].tolist() == [12, 24, 36, 48, 60, 72, 84]
    assert p._shift_k(0, 1)[:, 0].tolist() == [24, 48, 72] and p._shift_k(0, 2)[:, 0].tolist() == [48]


def _plans():
    out = [(n, inv, None) for n in range(1, 12) for inv in (False, True)]
    out += [(n, inv, None) for n in (12, 13, 17) for inv in (False, True)]
    out += [(n, False, b) for n, b in ((2, 1), (6, 3), (11, 1), (12, 2), (17, 3))]
    return out


@pytest.mark.parametrize("log_n,inverse,log_b", _plans())
def test_targeting_reaches_every_edge_class_at_every_step(log_n, inverse, log_b):
    """Runs the model forward from targeted inputs. At every targeted step, the state the model reaches is the requested
    one, and across the inputs every step sees every edge class of its kind: butterflies every class of PAIR_CLASSES,
    shifts every class of SHIFT_CLASSES, twiddle, pre-scale, post-twiddle and scale products every class of
    PRODUCT_CLASSES."""
    net = M.Network(log_n, inverse, log_b)
    rng = np.random.default_rng(log_n * 10 + inverse + 100 * (log_b or 0))
    coset = (1 << log_b) - 1 if log_b else 0
    for pi, ps in enumerate(net.passes):
        steps = M.spread_targets(net, pi, M.columns_for(net, pi))
        x, requested = net.target(pi, steps, rng, coset)
        seen, reached = {}, set()

        def observe(label, state, ops):
            p, i = label[:2]
            m = steps == i
            if p != pi or not m.any():
                return
            assert (state[coset][m] == requested[m]).all(), ("targeted state not reached", label)
            reached.add(i)
            seen[label] = M.classify(label[2], M.operands_at(ops, m, coset))

        net.forward(x, observe)
        assert reached == set(ps.targets()), (pi, sorted(set(ps.targets()) - reached))
        for label, classes in seen.items():
            want = {"bf": M.PAIR_CLASSES, "shift": M.SHIFT_CLASSES}.get(label[2], M.PRODUCT_CLASSES)
            assert set(want) <= classes, (label, set(want) - classes)


def test_targeting_a_later_pass_inverts_the_earlier_ones(oracle):
    # a pass-2 target of 2^12 is an input whose pass-2 state the oracle's own transform also reaches: the model's output
    # from it equals the oracle's, and the targeted butterflies of pass 2 sum to exactly p where requested
    net = M.Network(12)
    rng = np.random.default_rng(5)
    steps = np.full((1, net.nsub(1)), -1)
    bf0 = net.passes[1].steps.index(("bf", 0, 0))
    steps[0, ::3] = bf0
    x, requested = net.target(1, steps, rng)
    assert (net.forward(x)[0] == oracle.evaluate_poly(x[0])).all()
    sums = []

    def observe(label, state, ops):
        if label[:2] == (1, bf0):
            a, b = M.operands_at(ops, steps == bf0)
            sums.append(a.astype(object) + b.astype(object))
    net.forward(x, observe)
    assert any((s == M.P).any() for s in sums) and any((s == 2**64).any() for s in sums)
