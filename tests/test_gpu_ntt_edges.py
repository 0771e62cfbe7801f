"""The device's NTT, iNTT and LDE on inputs that reach the reduction edges inside its transform network: structured inputs
with closed-form transforms, and inputs that tests/ntt_model.py targets at every butterfly, shift, twiddle, pre-scale and
post-twiddle step of every plan (uniform random data reaches these edges with probability 2^-32 .. 2^-64 per operation).
Every output is compared bit for bit with the oracle (or with exact closed forms), and with the model where it is cheap."""
import numpy as np
import pytest

import ntt_model as M
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
P = wf.P
SIZES = list(range(1, 12)) + [12, 17, 22]


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    assert c.mem_stats()[0] == 0, "device buffers left live"
    c.close()


def _run(ctx, x, op, *args):
    m = ctx.mat_from_host_columns(x)
    out = getattr(m, op)(*args)
    got = out.to_columns() if op != "lde" else out.to_rows()
    m.free(); out.free()
    return got


# ---- every shift amount ----
def test_every_shift_amount_on_its_edges(ctx):
    import torch
    rng = np.random.default_rng(3)
    xs = {0, 1, 2, P - 1, P - 2, 2**32 - 1, 2**32, 0xFFFFFFFF00000000, 2**63}
    for k in range(97):
        xs |= {int(v) for v in M.shift_catalogue(k)}
    xs = np.array(sorted(xs) + [int(v) for v in rng.integers(0, P, 512, dtype=np.uint64)], dtype=np.uint64)
    n = xs.size
    a = torch.from_numpy(xs.view(np.int64)).cuda()
    out = torch.empty(97 * n, dtype=torch.int64, device="cuda")
    ctx.field_shifts_dev(a.data_ptr(), n, out.data_ptr())
    ctx.sync()
    got = out.cpu().numpy().view(np.uint64).reshape(97, n)
    for k in range(97):
        want = np.array([int(x) * pow(2, k, P) % P for x in xs], dtype=np.uint64)
        bad = np.nonzero(got[k] != want)[0]
        assert bad.size == 0, ("gl_mul_2exp", k, [hex(int(xs[i])) for i in bad[:4]])


# ---- structured inputs with closed-form transforms ----
def _structured(log_n):
    n = 1 << log_n
    w = M.root(log_n)
    cols, names = [], []

    def add(name, v):
        names.append(name); cols.append(np.asarray(v, dtype=np.uint64))
    for c in (0, P - 1, 2**32 - 1, 12345):
        add(("const", c), np.full(n, c))
    for k in sorted({0, n // 2, n - 1}):
        add(("impulse", k), np.eye(1, n, k, dtype=np.uint64)[0] * np.uint64(1))
    add(("alternating",), np.where(np.arange(n) & 1, P - 1, 0))
    for k in sorted({1, n // 2, n - 1}):
        add(("monomial evals", k), M.powers(pow(w, k, P), n))
    return names, np.stack(cols)


def _closed_form(name, log_n, inverse):
    n = 1 << log_n
    w = M.root(log_n)
    inv_n = pow(n, P - 2, P)
    out = np.zeros(n, dtype=np.uint64)
    if name[0] == "const":                    # all c
        out[0] = name[1] if inverse else name[1] * n % P
    elif name[0] == "impulse":                # e_k -> w^(+-jk) (/ n)
        k = name[1]
        out = M.powers(pow(w, (n - k) % n, P), n) if inverse else M.powers(pow(w, k, P), n)
        if inverse:
            out = M.fmul(out, np.uint64(inv_n))
    elif name[0] == "alternating":            # -[i odd]
        h = n // 2
        if inverse:
            out[0] = (P - 1) * pow(2, P - 2, P) % P
            out[h % n] = (out[h % n] + pow(2, P - 2, P)) % P
        else:
            out[0] = (P - h) % P
            out[h % n] = (out[h % n] + h) % P
    else:                                     # w^(jk) -> e_k, or n e_(-k)
        k = name[1]
        if inverse:
            out[k] = 1
        else:
            out[(n - k) % n] = n % P
    return out


@pytest.mark.parametrize("log_n", SIZES)
def test_structured_inputs(ctx, log_n):
    names, x = _structured(log_n)
    for inverse in (False, True):
        got = _run(ctx, x, "interpolate" if inverse else "evaluate")
        for i, name in enumerate(names):
            assert (got[i] == _closed_form(name, log_n, inverse)).all(), (log_n, inverse, name)
    # interpolating the evaluations of x^k gives exactly x^k: a cancels against p - a throughout the last layers
    n = 1 << log_n
    ks = sorted({k % n for k in (0, 1, 2, n // 3, n - 2, n - 1)})
    mono = np.stack([M.powers(pow(M.root(log_n), k, P), n) for k in ks])
    got = _run(ctx, mono, "interpolate")
    for i, k in enumerate(ks):
        assert (got[i] == np.eye(1, n, k, dtype=np.uint64)[0]).all(), (log_n, k)


# ---- targeted inputs ----
def _targeted(log_n, inverse, rng, passes=None, per_step=64, log_b=None, coset=0):
    net = M.Network(log_n, inverse, log_b)
    xs = []
    for pi in (range(len(net.passes)) if passes is None else passes):
        steps = M.spread_targets(net, pi, M.columns_for(net, pi, per_step))
        xs.append(net.target(pi, steps, rng, coset)[0])
    return net, np.concatenate(xs)


def _check_ntt(oracle, got, x, inverse, net=None):
    fn = oracle.interpolate_poly if inverse else oracle.evaluate_poly
    for c in range(x.shape[0]):
        assert (got[c] == fn(x[c])).all(), ("device != oracle", c)
    if net is not None:
        assert (got == net.forward(x)).all(), "device != model"


@pytest.mark.parametrize("log_n", SIZES)
def test_targeted_evaluate_and_interpolate(ctx, oracle, log_n):
    rng = np.random.default_rng(700 + log_n)
    for inverse in (False, True):
        if log_n == 22:     # one column per direction: the last pass forward, the first one inverse
            net, x = _targeted(log_n, inverse, rng, passes=[0 if inverse else 1], per_step=1)
        else:
            net, x = _targeted(log_n, inverse, rng)
        got = _run(ctx, x, "interpolate" if inverse else "evaluate")
        _check_ntt(oracle, got, x, inverse, net if log_n <= 17 else None)


@pytest.mark.parametrize("ncols", [1, 2, 3, 4, 5, 8, 9, 13])
@pytest.mark.parametrize("log_n", [6, 11, 12])
def test_targeted_segment_widths(ctx, oracle, log_n, ncols):
    # segment widths 1, 2, 4 and 8, and partly filled last segments: every T / chunks tile geometry
    rng = np.random.default_rng(ncols * 31 + log_n)
    for inverse in (False, True):
        net, x = _targeted(log_n, inverse, rng, per_step=8)
        x = x[rng.permutation(x.shape[0])[:ncols]] if x.shape[0] >= ncols else np.resize(x, (ncols, x.shape[1]))
        _check_ntt(oracle, _run(ctx, x, "interpolate" if inverse else "evaluate"), x, inverse, net)


@pytest.mark.parametrize("log_n", [12, 16, 20])
@pytest.mark.parametrize("log_b", [1, 2, 3])
def test_targeted_lde(ctx, oracle, log_n, log_b):
    # every step of the LDE's first pass of one coset, the coset pre-scale of round 0 and the post twiddle included;
    # through Mat.lde and through lde_into (the in-place, all-cosets y_in_out path)
    rng = np.random.default_rng(log_n * 8 + log_b)
    coset = (log_n + log_b) % (1 << log_b)
    net, x = _targeted(log_n, False, rng, passes=[0], per_step=16 if log_n < 20 else 1, log_b=log_b, coset=coset)
    want = oracle.lde_rows(x, 1 << log_b)
    assert (_run(ctx, x, "lde", log_b) == want).all()
    if log_n <= 16:
        assert (net.forward(x) == want.T).all()
    m = ctx.mat_from_host_columns(x)
    out = ctx.mat_from_host_columns(np.zeros((x.shape[0], x.shape[1] << log_b), dtype=np.uint64))
    m.lde_into(log_b, out)
    assert (out.to_rows() == want).all()
    m.free(); out.free()


@pytest.mark.parametrize("log_n", [4, 11, 12])
def test_targeted_interpolate_with_offset(ctx, oracle, log_n):
    rng = np.random.default_rng(log_n)
    _, x = _targeted(log_n, True, rng, per_step=16)
    got = _run(ctx, x, "interpolate_with_offset", 7)
    for c in range(x.shape[0]):
        assert (got[c] == oracle.interpolate_poly_with_offset(x[c], 7)).all()


@pytest.mark.parametrize("log_n", [5, 9, 12])
def test_targeted_ntt_dev_in_place(ctx, oracle, log_n):
    import torch
    rng = np.random.default_rng(50 + log_n)
    for inverse in (False, True):
        net, x = _targeted(log_n, inverse, rng, per_step=16)
        d = torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).cuda()
        ctx.ntt_dev(d.data_ptr(), log_n, x.shape[0], inverse)
        ctx.sync()
        _check_ntt(oracle, d.cpu().numpy().view(np.uint64), x, inverse, net)


@pytest.mark.parametrize("ncols", [3, 8, 11])
def test_targeted_trace_lde_from_host(ctx, oracle, ncols):
    # the column-chunked pipeline: chunks of a segment land at out_col0 > 0, the last chunk partly filled
    rng = np.random.default_rng(ncols)
    _, x = _targeted(12, True, rng, per_step=8)
    x = np.resize(x, (ncols, x.shape[1]))
    polys, lde = ctx.trace_lde_from_host(x, 2)
    want = oracle.interpolate_columns(x)
    assert (polys.to_columns() == want).all()
    assert (lde.to_rows() == oracle.lde_rows(want, 4)).all()
    polys.free(); lde.free()


@pytest.mark.parametrize("log_n,inverse,log_b", [(23, False, None), (24, True, None), (23, False, 1)])
def test_targeted_three_pass(ctx, oracle, log_n, inverse, log_b):
    # one column whose sub-transforms of the first pass (8 points) are targeted at every step, pre-scale and post twiddle
    # of the three-pass LDE included
    rng = np.random.default_rng(log_n)
    _, x = _targeted(log_n, inverse, rng, passes=[0], per_step=1, log_b=log_b, coset=1 if log_b else 0)
    if log_b:
        assert (_run(ctx, x, "lde", log_b) == oracle.lde_rows(x, 1 << log_b)).all()
    else:
        _check_ntt(oracle, _run(ctx, x, "interpolate" if inverse else "evaluate"), x, inverse)
