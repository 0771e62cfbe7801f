"""The device's hashers on inputs at the edges of their encodings: the Rescue S-box and MDS arithmetic on any 64-bit words
(wf_rescue_ops_dev) bit for bit against the exact model (rescue_model.py), the permutations and merges on states targeted at
every step boundary and at each of the Jive sum's three adds (wf_rescue_permute_dev), the row-hash, Merkle and FRI layer
kernels on inputs targeted at round 0, second sponge blocks aimed at absorb sums p - 1 and p, every hasher at every sponge
block edge, and merges of digests whose words are p or more."""
import numpy as np
import pytest

import dishonest as D
import rescue_model as M
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
P = M.P
ALL = [wf.HASH_BLAKE3_256, wf.HASH_RP64_256, wf.HASH_RPJIVE64_256, wf.HASH_BLAKE3_192, wf.HASH_SHA3_256]


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    assert c.mem_stats()[0] == 0, "device buffers left live"
    c.close()


def _dev(words):
    import torch
    return torch.from_numpy(np.ascontiguousarray(np.array(words, dtype=np.uint64)).view(np.int64)).cuda()


def _host(t):
    return [int(v) for v in t.cpu().numpy().view(np.uint64)]


def _weak_operands():
    rng = np.random.default_rng(17)
    words = {0, 1, 2, P - 1, P - 2, P, P + 1, 2**32 - 1, 2**32, 2**32 + 1, P - 2**32, 2**63, 2**64 - 1, 2**64 - 2,
             0xFFFFFFFF00000000, 0x00000000FFFFFFFF}
    found, _ = M.slot_targets()
    for xs in found.values():
        words |= set(xs)
    words |= {v + P for v in range(0, 40)} | {2**64 - 1 - v for v in range(40)}
    words = sorted(words) + [int(v) for v in rng.integers(0, 2**64, 480, dtype=np.uint64)]
    # MDS inputs whose 32-bit-half sums take the l < lo carry: all low halves 2^32 - 1, high halves with hi = -1 mod 2^32
    for h in (M.HASHERS[M.RP64], M.HASHERS[M.RPJIVE]):
        c0 = h.mat[0][0]
        hi0 = (-(sum(h.mat[0][1:]) * (2**32 - 1)) - 1) * pow(c0, -1, 2**32) % 2**32
        words += [(hi0 << 32) | (2**32 - 1)] + [2**64 - 1] * (h.w - 1)
    words += [2**64 - 1] * 24
    words += [0] * (-len(words) % 24)
    return words


def test_weak_arithmetic_on_any_words(ctx):
    import torch
    a = _weak_operands()
    n = len(a)
    b = a[7:] + a[:7]
    out = torch.empty(10 * n, dtype=torch.int64, device="cuda")
    ta, tb = _dev(a), _dev(b)   # held: a temporary's memory would be handed to the next allocation
    ctx.rescue_ops_dev(ta.data_ptr(), tb.data_ptr(), n, out.data_ptr())
    ctx.sync()
    got = _host(out)
    blk = lambda k: got[k * n:(k + 1) * n]   # noqa: E731
    for x, y, m, s, e in zip(a, b, blk(0), blk(1), blk(2)):
        assert m % P == x * y % P and m == M.mul_weak(x, y), ("gl_mul_weak", hex(x), hex(y), hex(m))
        assert s % P == x * x % P and s == M.mul_weak(x, x), ("gl_sqr_weak", hex(x), hex(s))
        assert e % P == pow(x, 7, P) and e == M.exp7(x), ("rp64_exp7", hex(x), hex(e))
    for k, g in enumerate([1, 2, 3, 4, 6]):
        for x, r in zip(a, blk(3 + k)):
            assert r % P == pow(x, M.INV7, P) and r == M.inv7(x), ("rp64_inv7_group", g, hex(x), hex(r))
    for hid, k in ((M.RP64, 8), (M.RPJIVE, 9)):
        h = M.HASHERS[hid]
        for i in range(0, n, h.w):
            s = a[i:i + h.w]
            want = [sum(c * v for c, v in zip(row, s)) % P for row in h.mat]
            assert blk(k)[i:i + h.w] == want == M.mds(h, s), ("mds", hid, i)


def _permute_check(ctx, oracle, hid, states, values):
    import torch
    w = M.HASHERS[hid].w
    n = len(states)
    out = torch.empty(n * (w + 8), dtype=torch.int64, device="cuda")
    ts, tv = _dev([v for s in states for v in s]), _dev(values)
    ctx.rescue_permute_dev(hid, ts.data_ptr(), tv.data_ptr(), n, out.data_ptr())
    ctx.sync()
    got = _host(out)
    perm = oracle.rp64_permute if hid == M.RP64 else oracle.rpjive_permute
    d = lambda ws: np.array(ws, dtype=np.uint64).tobytes()   # noqa: E731
    red = lambda ws: [x % P for x in ws]                     # noqa: E731
    for i, (s, v) in enumerate(zip(states, values)):
        assert got[i * w:(i + 1) * w] == [int(x) for x in perm(np.array(red(s), dtype=np.uint64))] == M.permute(hid, s), ("permute", i)
        m = got[n * w + 4 * i:n * w + 4 * i + 4]
        assert d(m) == oracle.merge(hid, d(red(s[:4])), d(red(s[4:8]))), ("merge", i)
        mi = got[n * (w + 4) + 4 * i:n * (w + 4) + 4 * i + 4]
        assert d(mi) == oracle.merge_with_int(hid, d(red(s[:4])), v), ("merge_with_int", i, hex(v))


@pytest.mark.parametrize("hid", [M.RP64, M.RPJIVE])
def test_permutation_on_targeted_states(ctx, oracle, hid):
    rng = np.random.default_rng(hid)
    states = [s for _, s in M.targeted_states(hid, rng)]
    vals = [0, 1, 5, P - 1, P, P + 1, 2**64 - 1, 2**63]
    _permute_check(ctx, oracle, hid, states, [vals[i % len(vals)] for i in range(len(states))])


def test_jive_sum_at_its_edges(ctx, oracle):
    # each of the three adds of the Jive sum at p and in [p, 2^64): the input pair through the input words, the output pair
    # backward from the round-6 output, the last add through the searched input (rescue_model.JIVE_LAST_ADD_INPUT)
    states = [s for _, s in M.jive_edge_states(np.random.default_rng(11))]
    log = M.Log()
    for s in states:
        M.jive(s, log)
    for kind in ("jive inputs", "jive outputs", "jive last"):
        assert log.hits.get((kind, "sum in [p, 2^64)")), kind
    _permute_check(ctx, oracle, M.RPJIVE, states, [P - 1] * len(states))


@pytest.mark.parametrize("hid", [M.RP64, M.RPJIVE])
def test_second_block_absorb_sums(ctx, oracle, hid):
    # rows of two blocks whose second block's absorb adds sum to p - 1 and p
    rows = np.array(M.two_block_rows(hid, np.random.default_rng(hid + 20), count=8), dtype=np.uint64)
    log = M.Log()
    for r in rows:
        M.hash_elements(hid, [int(v) for v in r], log)
    assert log.hits.get(("absorb", "sum p")) and log.hits.get(("absorb", "sum p - 1"))
    m = ctx.mat_from_host_columns(np.ascontiguousarray(rows.T))
    t = ctx.commit_rows(hid, m)
    assert (t.to_host()[0] == oracle.hash_rows(hid, rows)).all()
    t.free(); m.free()


@pytest.mark.parametrize("hid,d,nf", [(M.RP64, 1, 8), (M.RP64, 2, 4), (M.RPJIVE, 1, 4), (M.RPJIVE, 2, 2)])
def test_fri_layer_leaves_on_round0_targets(ctx, oracle, hid, d, nf):
    # FRI layer 0 hashes the nf evaluations at positions i, i + L / nf, ... of each row i (nf d words): evaluations laid out
    # so that those rows are the round-0 targets; the layer roots and the remainder are compared with the oracle's
    rng = np.random.default_rng(hid * 10 + nf)
    L, b = 1 << 10, 8
    rows = M.round0_rows(hid, rng, nf * d)
    ev = np.zeros((nf, L // nf, d), dtype=np.uint64)
    for i in range(L // nf):
        row = rows[i % len(rows)]
        for k in range(nf):
            ev[k, i] = row[k * d:(k + 1) * d]
    ev = ev.reshape(-1)
    want_roots, want_rem, _ = oracle.fri_build_layers(hid, ev, nf, 7, b, d)
    m = ctx.mat_from_host_columns(np.ascontiguousarray(ev.reshape(L, d).T))
    f, roots = ctx.fri_build_layers_default(hid, m, d, nf, 7, b)
    assert (roots == want_roots).all()
    assert (f.remainder() == want_rem).all()
    f.free(); m.free()


@pytest.mark.parametrize("hid", [M.RP64, M.RPJIVE])
def test_merge_of_digests_with_words_of_p_or_more(ctx, oracle, hid):
    # the reference reads a digest word w >= p as w - p (ElementDigest::read_from): the device's merges of such digests must
    # equal the merges of the reduced ones, on either side of the merge and in the merge_with_int seed
    rng = np.random.default_rng(40 + hid)
    w = M.HASHERS[hid].w
    states = []
    for k in range(64):
        s = [int(v) for v in rng.integers(0, 2**32 - 1, w, dtype=np.uint64)]
        s = [x + P if (k >> (j % 6)) & 1 else x for j, x in enumerate(s)]
        s[k % 8] = 2**64 - 1
        states.append(s)
    _permute_check(ctx, oracle, hid, states, [P - 1, P, 2**64 - 1, 3] * 16)


@pytest.mark.parametrize("hid", [M.RP64, M.RPJIVE])
def test_row_hash_kernels_on_round0_targets(ctx, oracle, hid):
    rng = np.random.default_rng(hid + 2)
    rate = 8 if hid == M.RP64 else 4
    for width in range(1, rate + 1):
        rows = np.array(M.round0_rows(hid, rng, width), dtype=np.uint64)
        rows = np.resize(rows, (max(8, 1 << (len(rows) - 1).bit_length()), width))
        want = oracle.hash_rows(hid, rows)
        m = ctx.mat_from_host_columns(np.ascontiguousarray(rows.T))
        t = ctx.commit_rows(hid, m)
        lv, nd = t.to_host()
        assert (lv == want).all(), width
        assert (nd == oracle.merkle_nodes(hid, want)).all(), width
        t.free()
        t = ctx.commit_rows(hid, m, partition_size=max(1, width // 2))
        assert (t.to_host()[0] == oracle.hash_rows(hid, rows, partition_size=max(1, width // 2))).all(), width
        t.free(); m.free()
        import torch
        dg = torch.empty(len(rows) * 32, dtype=torch.uint8, device="cuda")
        tr = _dev(rows.reshape(-1))
        ctx.hash_rows_dev(hid, tr.data_ptr(), len(rows), width, dg.data_ptr())
        ctx.sync()
        assert (dg.cpu().numpy().reshape(-1, 32) == want).all(), width


@pytest.mark.parametrize("log_leaves", [4, 15])
@pytest.mark.parametrize("hid", [M.RP64, M.RPJIVE])
def test_merkle_kernels_on_targeted_merges(ctx, oracle, hid, log_leaves):
    # leaf pairs that are targeted merge inputs: Rp64 merges see them as round-0 S-box inputs, RpJive merges control their
    # whole state, so every step of every round is reached. 2^15 leaves: more than 2^13 parents on the per-level kernel
    rng = np.random.default_rng(hid * 3 + log_leaves)
    states = [s[:8] for _, s in M.targeted_states(hid, rng)]
    if hid == M.RP64:
        found, _ = M.slot_targets()
        xs = M.SBOX_INPUTS + sorted({x for (s, _), v in found.items() if s.startswith("exp7") for x in v})
        states += [[xs[(k + j) % len(xs)] for j in range(8)] for k in range(0, len(xs), 8)]
    n = 1 << log_leaves
    leaves = np.array([states[i % len(states)] for i in range(n // 2)], dtype=np.uint64).reshape(n, 4)
    leaves = leaves.view(np.uint8).reshape(n, 32)
    t = ctx.tree_from_leaves(hid, leaves)
    _, nd = t.to_host()
    assert (nd == oracle.merkle_nodes(hid, leaves)).all()
    t.free()


@pytest.mark.parametrize("h", ALL)
def test_every_block_edge(ctx, oracle, h):
    # widths around the rates: Rp64 8, RpJive 4, SHA3-256 17 words, BLAKE3 a 1024-byte chunk of 128 words
    rows = 64
    for cols in list(range(1, 41)) + [63, 64, 65, 66, 127, 128, 129, 130, 136, 254, 255]:
        x = oracle.rand_elems((cols, rows), 1000 + cols + h)
        m = ctx.mat_from_host_columns(x)
        t = ctx.commit_rows(h, m)
        assert (t.to_host()[0] == oracle.hash_rows(h, np.ascontiguousarray(x.T))).all(), cols
        t.free(); m.free()
    # partition sizes on the SHA3 block, and merge_many messages of 16 and 20 words (4 and 5 partition digests)
    for cols, psize in ((34, 17), (51, 17), (68, 17), (85, 17), (68, 34), (136, 34), (40, 10), (20, 4), (25, 5)):
        x = oracle.rand_elems((cols, rows), 7 * cols + psize + h)
        m = ctx.mat_from_host_columns(x)
        t = ctx.commit_rows(h, m, partition_size=psize)
        assert (t.to_host()[0] == oracle.hash_rows(h, np.ascontiguousarray(x.T), partition_size=psize)).all(), (cols, psize)
        t.free(); m.free()


@pytest.mark.parametrize("ext", [1, 2, 3])
@pytest.mark.parametrize("h", ALL)
def test_verifier_refuses_words_of_p_or_more(ctx, h, ext):
    # the oracle's verdicts (test_oracle_noncanonical_proofs.py pins them) from the device, in one batch with the honest proof
    cases = D.noncanonical_cases(h, ext)
    pv = D.Prover("perm_rap", 64)
    want = [pv.oracle_verdict(c.proof, h) for c in cases]
    got = [int(v) for v in ctx.verify_air_batch([c.desc for c in cases], [c.proof for c in cases], h)]
    assert ctx.mem_stats()[0] == 0
    wrong = [(c.name, g, w) for c, g, w in zip(cases, got, want) if g != w or (c.want is not None and g != c.want)]
    assert not wrong, wrong
