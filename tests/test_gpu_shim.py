"""The drop-in boundary exercised the way a reference-side binding would use it.

include/winterfell_b200.hpp mirrors the reference's prover plugin types (TraceLde, ConstraintEvaluator,
ConstraintCommitment, FriProver, ProverChannel; prover/src/lib.rs:125-223) over the C ABI, and its
generate_proof() is the call-for-call double of Prover::generate_proof (lib.rs:282-492) with the transcript
and the proof serializer on the host side of the boundary. The driver (tests/shim/generate_proof_main.cpp)
is plain g++ code linked against libwinterfell_b200.so; its proofs must be byte-identical to the
one-call entry points and to the oracle prover, and the oracle verifier must accept them."""
import os
import subprocess
import sys

import numpy as np
import pytest

import airs
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu

DRIVER = os.path.join(os.path.dirname(wf.__file__), "_build", "generate_proof_main")


def run_double(tmp_path, desc, trace, opts, mont=0, aux=None):
    if not os.path.exists(DRIVER):
        pytest.fail(f"{DRIVER} missing: run winterfell_b200/build.sh")
    n = trace.shape[1]
    words = [np.array([n.bit_length() - 1, mont], dtype=np.uint64), opts.astype(np.uint64),
             np.array([desc.size], dtype=np.uint64), desc, np.ascontiguousarray(trace, dtype=np.uint64).ravel()]
    if aux is None:
        words.append(np.array([0], dtype=np.uint64))
    else:
        rand, cols = aux
        words += [np.array([1], dtype=np.uint64), rand.ravel(), cols.ravel()]
    inp, out = tmp_path / "in.bin", tmp_path / "proof.bin"
    np.concatenate(words).tofile(inp)
    r = subprocess.run([DRIVER, str(inp), str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return out.read_bytes()


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("name,log_n,ext,h,batch", [
    ("fib", 7, 1, wf.HASH_RP64_256, 0),           # the reference's fib_small test shape
    ("fib", 10, 2, wf.HASH_BLAKE3_256, 1),
    ("mulfib2", 9, 3, wf.HASH_BLAKE3_256, 2),
    ("periodic_mix", 11, 1, wf.HASH_BLAKE3_256, 0),
    ("periodic_mix", 8, 3, wf.HASH_RP64_256, 1),
    ("sequence_mix", 9, 2, wf.HASH_BLAKE3_256, 0),
])
def test_cpp_generate_proof_double(ctx, oracle, tmp_path, name, log_n, ext, h, batch):
    n = 1 << log_n
    desc, trace = airs.fib_small_x(2, n) if name == "fib" else getattr(airs, name)(n)
    opts = oracle.make_opts(num_queries=20, blowup=8, grinding=3, ext=ext, folding=4, rem_max_deg=7, batch_c=batch, batch_d=batch, hash_id=h)
    got = run_double(tmp_path, desc, trace, opts)
    assert got == ctx.prove_air(desc, trace, opts)
    assert got == oracle.prove_air(desc, trace, opts)
    assert oracle.verify_air(desc, got, h) == 0


def test_cpp_double_with_partitions(ctx, oracle, tmp_path):
    # new_trace_lde / build_constraint_commitment take the PartitionOptions (prover/src/lib.rs:187,220): the C++ mirror passes
    # them to wf_commit_rows_partitioned / wf_composition_commit_partitioned
    desc, trace = airs.fib_small_x(4, 512)
    opts = oracle.make_opts(num_queries=20, grinding=3, ext=3, folding=4, rem_max_deg=7, num_partitions=4, hash_rate=8)
    got = run_double(tmp_path, desc, trace, opts)
    assert got == ctx.prove_air(desc, trace, opts)
    assert got == oracle.prove_air(desc, trace, opts)
    assert oracle.verify_air(desc, got, 0) == 0


def test_cpp_double_montgomery_trace(ctx, oracle, tmp_path):
    # a Rust caller hands over &[BaseElement] memory = Montgomery words (math/src/field/f64/mod.rs:57-64)
    desc, trace = airs.mulfib2(256)
    opts = oracle.make_opts(num_queries=16, blowup=8, ext=2, folding=4, rem_max_deg=7)
    to_m = np.vectorize(lambda v: oracle.to_mont(int(v)), otypes=[np.uint64])
    assert run_double(tmp_path, desc, to_m(trace), opts, mont=1) == oracle.prove_air(desc, trace, opts)


@pytest.mark.parametrize("ext", [1, 3])
def test_cpp_double_aux_segment(ctx, oracle, tmp_path, ext):
    desc, trace, builder = airs.perm_rap(256)
    opts = oracle.make_opts(num_queries=20, blowup=8, grinding=2, ext=ext, folding=4, rem_max_deg=7, batch_c=2, batch_d=2)
    seen = {}

    def recording(rand):
        seen["rand"] = rand.copy()
        seen["cols"] = builder(rand)
        return seen["cols"]

    want = oracle.prove_air_aux(desc, trace, opts, recording, airs.PERM_RAP_AUX_WIDTH, 2)
    got = run_double(tmp_path, desc, trace, opts, aux=(seen["rand"], seen["cols"]))
    assert got == want
    assert oracle.verify_air(desc, got) == 0


def test_stepwise_python_matches_one_call(ctx, oracle):
    """The same steps through the Python mirror of the ABI (host transcript = the oracle's RandomCoin):
    every intermediate the reference's traits hand back is reachable and consistent."""
    n, log_n, ext, h = 512, 9, 2, wf.HASH_BLAKE3_256
    desc, trace = airs.periodic_mix(n)
    opts = oracle.make_opts(num_queries=12, blowup=8, ext=ext, folding=4, rem_max_deg=7, hash_id=h)
    m = ctx.mat_from_host_columns(trace)
    polys = m.interpolate()
    lde = polys.lde(3)
    tree = ctx.commit_rows(h, lde)
    # TraceLde::read_main_trace_frame_into: rows (s, s + blowup mod N) of the LDE
    fr = lde.read_rows(np.array([5, 13], dtype=np.uint64))
    want = oracle.lde_rows(oracle.interpolate_columns(trace), 8)
    assert (fr[0] == want[5]).all() and (fr[1] == want[13]).all()
    # constraint evaluation with fixed coefficients: every CE row equals the oracle prover's value from the same frames
    ntr, nas = 3, 5
    coeffs = oracle.rand_elems((ntr + nas, ext), 11)
    comp = ctx.eval_constraints(desc, log_n, 8, ext, lde, None, coeffs)
    assert comp.rows == n * 4 and comp.cols == ext
    rows = np.arange(n * 4, dtype=np.uint64)
    ls = rows.astype(np.int64) << 1                     # ce_blowup 4, blowup 8
    got = comp.to_rows()
    assert (got == oracle.eval_constraint_rows(desc, n, 8, ext, coeffs, None, rows, want[ls], want[(ls + 8) % (8 * n)])).all()
    comp2 = ctx.eval_constraints(desc, log_n, 8, ext, lde, None, coeffs)
    assert (got == comp2.to_rows()).all()
    cpolys, clde, ctree = ctx.composition_commit(h, comp, log_n, 8, ext, 3)
    assert cpolys.rows == n and cpolys.cols == 3 * ext and clde.rows == 8 * n
    # the composition columns, evaluated at z, recombine to the CE-domain polynomial: H(z) = sum_i z^(i n) H_i(z)
    z = oracle.rand_elems((ext,), 5)
    zg = oracle.ext_mul(z, np.array([oracle.root_of_unity(log_n)] + [0] * (ext - 1), dtype=np.uint64))
    q0, q1 = ctx.evaluate_at(cpolys, ext, ext, z, zg)
    t0, _ = ctx.evaluate_at(polys, ext, 1, z, zg)
    for j in range(trace.shape[0]):
        assert (t0[j] == oracle.eval_poly_at(oracle.interpolate_columns(trace)[j], z, 1)).all()
    deep = ctx.deep_compose(ext, lde, None, clde, log_n, z, oracle.rand_elems((3 + 3, ext), 3),
                            np.concatenate([t0, q0]), np.concatenate([ctx.evaluate_at(polys, ext, 1, z, zg)[1], q1]))
    assert deep.rows == 8 * n and deep.cols == ext
    # DEEP composition of consistent inputs is a polynomial of degree <= n - 2 (composer/mod.rs:171-180)
    dcoef = deep.interpolate_with_offset(7).to_rows()
    assert dcoef[: n - 1].any() and not dcoef[n - 1:].any()
    for o in (m, polys, lde, comp, comp2, cpolys, clde, deep):
        o.free()
    for t in (tree, ctree):
        t.free()
