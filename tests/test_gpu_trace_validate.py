"""wf_trace_validate and wf_ctx_set_validation on the device:
- the report, the first failing step of every transition constraint and both degree lists equal the CPU restatement's
  (tests/trace_validate_ref.py) for every fixture of tests/airs.py and every planted violation of
  tests/test_trace_validate_oracle.py, over ext 1 / 2 / 3, host, device and Montgomery traces, host aux columns and aux build
  descriptions (a wrong init or term included), 2^3 to 2^13 rows, one and two exemptions; one constructed case at 2^18 rows;
- with validation on, proofs of valid traces are byte-identical to the proofs with it off, for wf_prove_air, _aux, _aux_dyn,
  _aux_built and wf_prove_air_batch; a violation refuses each of them with the reference's message, writes nothing and leaves
  no device buffer live; wf_eval_constraints refuses a wrongly declared degree."""
import numpy as np
import pytest

import airs
import aux_builds as ab
import trace_validate_ref as R
import winterfell_b200 as wf
from test_trace_validate_oracle import cycled, fixtures, planted, redeclared

pytestmark = pytest.mark.gpu
P = wf.P


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def same(got, want):
    for k in ("kind", "index", "step", "column", "first_failing_step", "expected_degrees", "actual_degrees", "msg"):
        assert got[k] == want[k], (k, got[k], want[k])


def to_mont(a):
    L = wf.lib()
    return np.vectorize(lambda v: L.wf_host_canonical_to_mont(int(v)), otypes=[np.uint64])(a)


def rand_for(ext, seed=77):
    from oracle import oracle as O
    return O.rand_elems((2, ext), seed)


@pytest.mark.parametrize("ext", [1, 2, 3])
@pytest.mark.parametrize("n", [8, 64, 1 << 13])
@pytest.mark.parametrize("i", range(6))
def test_fixtures_match_the_restatement(ctx, oracle, ext, n, i):
    if n == 1 << 13 and i not in (0, 5):
        pytest.skip("2^13 rows: one single-segment and one two-segment fixture")
    name, desc, tr, aux, rand = fixtures(n, ext)[i]
    want = R.validate(desc, tr, aux, rand, ext)
    same(ctx.trace_validate(desc, tr, ext, rand=rand, aux=aux), want)
    assert ctx.mem_stats()[0] == 0


@pytest.mark.parametrize("ext", [1, 2, 3])
@pytest.mark.parametrize("i", range(11))
def test_planted_violations_match_the_restatement(ctx, oracle, ext, i):
    name, desc, tr, aux, rand, _ = planted()[i]
    if aux is not None and ext != 2:   # the case's changed cells, in columns built for this extension degree
        n = tr.shape[1]
        cells = {(int(c), int(s)) for c, s, _ in np.argwhere(aux != airs.perm_rap(n)[2](rand))}
        rand = rand_for(ext, 5)
        aux = airs.perm_rap(n)[2](rand)
        for c, s in cells:
            aux[c, s, 0] = (int(aux[c, s, 0]) + 1) % P
    want = R.validate(desc, tr, aux, rand, ext)
    assert want["kind"] != R.VALID or name == "exempt_rows"
    same(ctx.trace_validate(desc, tr, ext, rand=rand, aux=aux), want)


def test_device_and_montgomery_traces(ctx, oracle):
    import torch
    for case in (planted()[3], planted()[6], planted()[9]):
        name, desc, tr, aux, rand, _ = case
        want = R.validate(desc, tr, aux, rand, 2)
        dev = torch.from_numpy(tr.view(np.int64)).cuda().contiguous()
        same(ctx.trace_validate(desc, dev.data_ptr(), 2, rand=rand, aux=aux, n=tr.shape[1]), want)
        got = ctx.trace_validate(desc, to_mont(tr), 2, rand=rand, aux=None if aux is None else to_mont(aux), mont=True)
        same(got, want)
        assert ctx.mem_stats()[0] == 0


def wrong_build(kind):
    """perm_rap's build description with the running product's init 2 ("init") or the counter's term 2 ("term")."""
    B = ab.AuxBuild(3, airs.PERM_RAP_AUX_WIDTH, 1, 2)
    p = B.column(ab.RUNNING_PRODUCT, (2 if kind == "init" else 1, 0, 0))
    p.num(p.add(p.cur(0), p.rnd(0)))
    p.den(p.add(p.cur(2), p.rnd(0)))
    q = B.column(ab.RUNNING_SUM)
    q.num(q.mul(q.mul(q.rnd(1), q.per(0)), q.mul(q.cur(1), q.acur(0))))
    c = B.column(ab.RUNNING_SUM, (5, 0, 0))
    c.num(c.const(2 if kind == "term" else 1))
    return B.build()


@pytest.mark.parametrize("ext", [1, 2, 3])
@pytest.mark.parametrize("build", ["right", "init", "term"])
def test_aux_build_descriptions(ctx, oracle, ext, build):
    n = 64
    desc, tr, _ = airs.perm_rap(n)
    rand = rand_for(ext)
    b = ab.perm_rap_build() if build == "right" else wrong_build(build)
    aux = ab.reference(desc, b, tr, rand)
    want = R.validate(desc, tr, aux, rand, ext)
    assert (want["kind"] == R.VALID) == (build == "right")
    assert want["kind"] in (R.VALID, R.AUX_ASSERTION, R.AUX_TRANSITION)
    same(ctx.trace_validate(desc, tr, ext, rand=rand, aux_build=b), want)
    assert ctx.mem_stats()[0] == 0


def test_degree_declarations(ctx, oracle):
    n = 256
    d, t = airs.mulfib2(n)
    f, ft = airs.fib_small_x(1, n)
    for desc, tr in ((redeclared(lambda: d, [(1, []), (2, [])]), t), (redeclared(lambda: f, [(1, []), (2, [])]), ft),
                     cycled(n, 4), cycled(n, 8), airs.periodic_mix(n), airs.periodic_mix(n, 16)):
        for ext in (1, 3):
            same(ctx.trace_validate(desc, tr, ext), R.validate(desc, tr, None, None, ext))


def test_large_trace_constructed(ctx, oracle):
    # FibSmall x 4 at 2^18 rows: valid, then one changed cell whose first failing constraint and step follow from x2' = x2 + x3
    n = 1 << 18
    desc, tr = airs.fib_small_x(4, n)
    rep = ctx.trace_validate(desc, tr, 3)
    assert rep["kind"] == wf.VALID and rep["expected_degrees"] == rep["actual_degrees"] == [0] * 8
    t1 = tr.copy()
    t1[2, 200001] = (int(tr[2, 200001]) + 1) % P
    rep = ctx.trace_validate(desc, t1, 3, check_degrees=False)
    assert (rep["kind"], rep["index"], rep["step"]) == (wf.VIOLATION_MAIN_TRANSITION, 2, 200000)
    assert rep["first_failing_step"] == [None, None, 200000, 200000, None, None, None, None]
    assert rep["msg"] == "main transition constraint 2 did not evaluate to ZERO at step 200000"
    assert ctx.mem_stats()[0] == 0


# ---- the switch in the provers ----
def opts(ext, blowup=8):
    from oracle import oracle as O
    return O.make_opts(num_queries=20, blowup=blowup, grinding=0, ext=ext, folding=4, rem_max_deg=7)


def with_validation(ctx, fn):
    ctx.set_validation(1)
    try:
        return fn()
    finally:
        ctx.set_validation(0)


@pytest.mark.parametrize("ext", [1, 2, 3])
def test_valid_proofs_are_unchanged(ctx, oracle, ext):
    n = 64
    for desc, tr in (airs.fib_small_x(2, n), airs.mulfib2(n), airs.sequence_mix(n), airs.rescue_like(n)):
        o = opts(ext)
        off = ctx.prove_air(desc, tr, o)
        assert with_validation(ctx, lambda: ctx.prove_air(desc, tr, o)) == off
        assert ctx.prove_air(desc, tr, o) == off
    desc, tr, builder = airs.perm_rap(n)
    o = opts(ext)
    off = ctx.prove_air_aux(desc, tr, o, builder, airs.PERM_RAP_AUX_WIDTH, 2)
    assert with_validation(ctx, lambda: ctx.prove_air_aux(desc, tr, o, builder, airs.PERM_RAP_AUX_WIDTH, 2)) == off
    assert with_validation(ctx, lambda: ctx.prove_air_aux_built(desc, ab.perm_rap_build(), tr, o)) == off
    dd, dtr, db = airs.perm_rap(n, dyn_last_q=True)
    off = ctx.prove_air_aux_dyn(dd, dtr, o, db, db.values_fn, airs.PERM_RAP_AUX_WIDTH, 2, db.num_values)
    assert with_validation(ctx, lambda: ctx.prove_air_aux_dyn(dd, dtr, o, db, db.values_fn, airs.PERM_RAP_AUX_WIDTH, 2,
                                                              db.num_values)) == off
    descs, trs = zip(*(airs.fib_small_x(2, n) for _ in range(3)))
    off = ctx.prove_air_batch(list(descs), list(trs), o)
    assert with_validation(ctx, lambda: ctx.prove_air_batch(list(descs), list(trs), o)) == off
    assert ctx.mem_stats()[0] == 0


def refused(ctx, fn, msg):
    with pytest.raises(wf.WfError) as e:
        with_validation(ctx, fn)
    assert msg in str(e.value), str(e.value)
    assert ctx.mem_stats()[0] == 0


def test_violations_refuse_every_entry_point(ctx, oracle):
    n, o = 32, opts(2)
    for name, desc, tr, aux, rand, want in planted():
        if want[0] == R.VALID:
            continue
        msg = R.check_trace(desc, tr, aux, rand, 2)["msg"]
        if aux is None:
            refused(ctx, lambda: ctx.prove_air(desc, tr, o), msg)
            if name == "main_transition":   # a batch names the refused proof
                good = airs.fib_small_x(2, n)[1]
                with pytest.raises(wf.WfError) as e:
                    with_validation(ctx, lambda: ctx.prove_air_batch([desc, desc], [good, tr], o))
                assert str(e.value).startswith("error -2: proof 1: ") and msg in str(e.value)
                assert ctx.mem_stats()[0] == 0
        else:
            # the same cells planted into the columns the prover's transcript draws its random elements for
            def planted_builder(r, aux=aux, rand=rand):
                full, ref = airs.perm_rap(n)[2](r), airs.perm_rap(n)[2](rand)
                return np.where(aux != ref, aux, full)
            with pytest.raises(wf.WfError) as e:
                with_validation(ctx, lambda: ctx.prove_air_aux(desc, tr, o, planted_builder, airs.PERM_RAP_AUX_WIDTH, 2))
            kind = {R.AUX_ASSERTION: "trace does not satisfy assertion aux_trace(", R.AUX_TRANSITION: "auxiliary transition constraint",
                    R.MAIN_TRANSITION: "main transition constraint"}[want[0]]
            assert kind in str(e.value)
            assert ctx.mem_stats()[0] == 0
    # aux build descriptions: a wrong init surfaces as an aux assertion, in the single and the batch entry point
    desc, tr, _ = airs.perm_rap(n)
    refused(ctx, lambda: ctx.prove_air_aux_built(desc, wrong_build("init"), tr, o), "trace does not satisfy assertion aux_trace(0, 0)")
    refused(ctx, lambda: ctx.prove_air_batch([desc], [tr], o, aux_build=wrong_build("term")), "proof 0: trace does not satisfy assertion aux_trace(2, 1)")
    # the degree check after constraint evaluation: periodic_mix over-declares two constraints
    d, t = airs.periodic_mix(n)
    refused(ctx, lambda: ctx.prove_air(d, t, o), "transition constraint degrees didn't match")


def test_eval_constraints_refuses_a_wrong_degree(ctx, oracle):
    n, log_b = 64, 3
    d, t = airs.fib_small_x(1, n)
    high = redeclared(lambda: d, [(1, []), (2, [])])
    m = ctx.mat_from_host_columns(t)
    polys = m.interpolate()
    lde = polys.lde(log_b)
    m.free()
    polys.free()
    coeffs = oracle.rand_elems((8, 2), 3)
    ok = with_validation(ctx, lambda: ctx.eval_constraints(d, 6, 8, 2, lde, None, coeffs))
    ok.free()
    with pytest.raises(wf.WfError) as e:
        with_validation(ctx, lambda: ctx.eval_constraints(high, 6, 8, 2, lde, None, coeffs))
    assert "transition constraint degrees didn't match" in str(e.value)
    lde.free()
    assert ctx.mem_stats()[0] == 0


def test_switch_off_launches_unchanged(ctx, oracle):
    desc, tr = airs.fib_small_x(2, 256)
    o = opts(2)
    ctx.prove_air(desc, tr, o)
    l0 = ctx.launches
    ctx.prove_air(desc, tr, o)
    off = ctx.launches - l0
    with_validation(ctx, lambda: ctx.prove_air(desc, tr, o))
    on = ctx.launches - l0 - off
    l1 = ctx.launches
    ctx.prove_air(desc, tr, o)
    assert ctx.launches - l1 == off and on > off
