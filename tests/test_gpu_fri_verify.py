"""wf_fri_verify_batch (FriVerifier::new + verify for a batch of standalone FRI proofs) against the CPU restatement's
wfr_fri_verify (tests/fri_ref.cpp), and wf_fri_build_proof against wfr_fri_build_proof: proof bytes, verdicts on honest, dishonest, byte-flipped and re-seeded
proofs, a mixed batch, launch counts and device memory."""
import ctypes as C

import numpy as np
import pytest

import winterfell_b200 as wf
import fri_cases as F
from fri_cases import HASHES, SHAPES, Case, default_positions, truncating_degree
from oracle import oracle as o

pytestmark = pytest.mark.gpu
V = F.fri_verdict


@pytest.fixture(scope="module")
def ctx():
    c = wf.Context(0)
    yield c
    c.close()


def device_proof(ctx, c, positions=None):
    """wf_fri_build_layers_default_channel + wf_fri_build_proof on the case's codeword: (proof bytes, roots)."""
    m = ctx.mat_from_host_columns(np.ascontiguousarray(c.ev.T))
    f, roots = ctx.fri_build_layers_default(c.h, m, c.d, c.nf, c.rem, c.blowup)
    proof = f.build_proof(c.pos if positions is None else positions)
    f.free()
    m.free()
    return proof, roots


def verify_batch(ctx, c, items, max_deg=None):
    """items: (proof, commitments, evaluations, coin seed) tuples verified in one call with the case's shape and positions."""
    return ctx.fri_verify_batch(c.h, c.d, c.nf, c.rem, c.blowup, c.max_deg if max_deg is None else max_deg, [it[0] for it in items],
                                [it[1] for it in items], [c.pos] * len(items), [it[2] for it in items], [it[3] for it in items])


def oracle_verdicts(c, items, max_deg=None):
    return [c.verify(proof=p, cm=cm, evals=ev, coin_seed=s, max_deg=max_deg) for p, cm, ev, s in items]


@pytest.mark.parametrize("h", HASHES)
@pytest.mark.parametrize("nf,rem", SHAPES)
@pytest.mark.parametrize("d", [1, 2, 3])
def test_build_proof_bytes(ctx, h, nf, rem, d):
    # the first direct test of wf_fri_build_proof: the FriProof bytes of the oracle's FriProver, and accepted on the device
    c = Case(h, d, nf, rem)
    proof, roots = device_proof(ctx, c)
    assert (roots == c.cm).all()
    assert proof == c.proof
    assert verify_batch(ctx, c, [(proof, roots, c.evals, None)]) == [F.FRI_VERIFY_ACCEPT]


def dishonest_items(c):
    """Proofs of the case's shape and positions with their oracle-built commitments: honest, wrong caller evaluations, every
    tamper, commitments changed, partition bytes rewritten."""
    items = [(c.proof, c.cm, c.evals, None)]
    for k in range(c.d):   # InvalidLayerFolding(0) from one coordinate of one evaluation, the last one included
        ev = c.evals.copy()
        ev[5, k] = (int(ev[5, k]) + 1) % o.P
        items.append((c.proof, c.cm, ev, None))
    for depth in sorted({1, c.nl - 1}):
        row = int(c.pos[1]) % c.layer_len(depth)
        t = c.tampered([o.tamper(o.FRI_LAYER, depth, row, (7,) * c.d)])
        items.append((t.proof, t.cm, c.evals, None))
    rn = c.layer_len(c.nl) // c.blowup
    for tp in ([o.tamper(o.REMAINDER_LONG, rn)], [o.tamper(o.REMAINDER, 0, delta=(1,) * c.d)], [o.tamper(o.FRI_LAYER, 0, int(c.pos[2]))]):
        t = c.tampered(tp)
        items.append((t.proof, t.cm, c.evals, None))
    cm = c.cm.copy()
    cm[-1] = 0xA5   # the remainder commitment is never compared: accepted
    items.append((c.proof, cm, c.evals, None))
    cm = c.cm.copy()
    cm[0, 0] ^= 0x10
    items.append((c.proof, cm, c.evals, None))
    for k in (1, 2, 5, 33, 63, 64, 200):
        p = bytearray(c.proof)
        p[-1] = k
        items.append((bytes(p), c.cm, c.evals, None))
    return items


@pytest.mark.parametrize("h", [o.BLAKE3, o.RP64, o.BLAKE3_192])
@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("nf,rem", [(2, 7), (4, 31), (16, 7)])
def test_verdicts_match_oracle(ctx, h, d, nf, rem):
    c = Case(h, d, nf, rem, log_n=10)
    items = dishonest_items(c)
    want = oracle_verdicts(c, items)
    assert want[0] == F.FRI_VERIFY_ACCEPT and want[-9] == F.FRI_VERIFY_ACCEPT
    assert V(F.FRI_VERIFY_INVALID_LAYER_FOLDING, 1) in want and F.FRI_VERIFY_REMAINDER_DEGREE_MISMATCH in want
    assert verify_batch(ctx, c, items) == want
    m, layer = truncating_degree(c.n, nf, c.nl)
    got = verify_batch(ctx, c, items[:3], max_deg=m)
    assert got == oracle_verdicts(c, items[:3], max_deg=m) == [V(F.FRI_VERIFY_DEGREE_TRUNCATION, layer)] * 3


@pytest.mark.parametrize("h,d", [(o.BLAKE3, 2), (o.RP64, 1), (o.SHA3, 3)])
def test_byte_flips(ctx, h, d):
    # every single-byte flip of an honest proof, in one batch
    c = Case(h, d, 4, 3, log_n=6, log_b=2, num_queries=6)
    items = []
    for i in range(len(c.proof)):
        p = bytearray(c.proof)
        p[i] ^= 1 << (i % 8)
        items.append((bytes(p), c.cm, c.evals, None))
    items += [(c.proof[:-1], c.cm, c.evals, None), (c.proof + b"\1", c.cm, c.evals, None), (c.proof, c.cm, c.evals, None)]
    want = oracle_verdicts(c, items)
    assert all(v != F.FRI_VERIFY_ACCEPT for v in want[:-1]) and want[-1] == F.FRI_VERIFY_ACCEPT
    assert verify_batch(ctx, c, items) == want


@pytest.mark.parametrize("h,d,nf", [(o.BLAKE3, 1, 4), (o.RP64, 3, 2), (o.RPJIVE, 2, 8)])
def test_coin_seed(ctx, h, d, nf):
    # a proof whose transcript starts from another coin: wf_fri_build_layers with callbacks that drive the oracle's coin from
    # that seed; accepted under its seed, refused under the default one
    c = Case(h, d, nf, 7, log_n=10)
    seed = bytes((7 * i + 3) % 256 for i in range(32))
    coin = o.RandomCoin(h)
    C.memmove(coin.c.seed, seed, 32)
    roots = []

    def commit(_user, root):
        r = bytes(root[:32])
        roots.append(r)
        coin.reseed(r)

    def draw(_user, out):
        a = coin.draw(d)
        for k in range(d):
            out[k] = int(a[k])

    cf, df = wf.FRI_COMMIT_FN(commit), wf.FRI_DRAW_FN(draw)
    m = ctx.mat_from_host_columns(np.ascontiguousarray(c.ev.T))
    fh = C.c_void_p()
    ctx.check(ctx.L.wf_fri_build_layers(ctx.h, h, m.h, d, nf, 7, c.blowup, cf, df, None, C.byref(fh)))
    f = wf.Fri(ctx, fh, d)
    cm = np.frombuffer(b"".join(roots), dtype=np.uint8).reshape(-1, 32)
    pos = coin.draw_integers(32, c.N, 0)
    proof = f.build_proof(pos)
    f.free()
    m.free()
    ev = c.ev[pos.astype(np.int64)]
    args = (h, d, nf, 7, c.blowup, c.max_deg)
    got = ctx.fri_verify_batch(*args, [proof] * 3, [cm] * 3, [pos] * 3, [ev] * 3, [seed, None, bytes(32)])
    want = [F.fri_verify(*args, proof, cm, pos, ev, s) for s in (seed, None, bytes(32))]
    assert got == want
    assert want[0] == F.FRI_VERIFY_ACCEPT and want[1] != F.FRI_VERIFY_ACCEPT and want[2] != F.FRI_VERIFY_ACCEPT
    assert ctx.fri_verify_batch(*args, [proof], [cm], [pos], [ev], None) == [want[1]]


def test_mixed_batch(ctx):
    # 1024 proofs of one shape, dishonest ones at scattered indices: each verdict is the one the proof gets alone
    base = [Case(o.BLAKE3, 3, 4, 31, log_n=10, seed=s) for s in (1, 2, 3)]
    c = base[0]
    rn = c.layer_len(c.nl) // c.blowup
    bad = {
        5: c.tampered([o.tamper(o.FRI_LAYER, 2, int(c.pos[0]) % c.layer_len(2), (1, 2, 3))]),
        131: c.tampered([o.tamper(o.REMAINDER_LONG, rn)]),
        512: c.tampered([o.tamper(o.REMAINDER, 1, delta=(0, 0, 1))]),
    }
    items, want = [], []
    for j in range(1024):
        if j in bad:
            t = bad[j]
            items.append((t.proof, t.cm, c.evals, None, c.pos))
        elif j in (77, 1023):   # someone else's evaluations
            items.append((c.proof, c.cm, base[1].ev[c.pos.astype(np.int64)], None, c.pos))
        elif j == 600:
            p = bytearray(c.proof)
            p[len(p) // 3] ^= 4
            items.append((bytes(p), c.cm, c.evals, None, c.pos))
        else:
            b = base[j % 3]
            items.append((b.proof, b.cm, b.evals, None, b.pos))
    for p, cm, ev, s, pos in items:
        want.append(F.fri_verify(c.h, 3, 4, 31, c.blowup, c.max_deg, p, cm, pos, ev, s))
    args = (c.h, 3, 4, 31, c.blowup, c.max_deg)
    got = ctx.fri_verify_batch(*args, *[[it[k] for it in items] for k in (0, 1, 4, 2)])
    assert got == want
    assert sum(v != F.FRI_VERIFY_ACCEPT for v in want) == 6
    for j in (5, 77, 131, 512, 600, 1023, 1022):
        p, cm, ev, s, pos = items[j]
        assert ctx.fri_verify_batch(*args, [p], [cm], [pos], [ev]) == [want[j]], j


def test_launch_count_does_not_depend_on_batch(ctx):
    c = Case(o.RP64, 2, 4, 31, log_n=12)
    counts = []
    for b in (1, 256):
        before = ctx.launches
        assert ctx.fri_verify_batch(c.h, 2, 4, 31, c.blowup, c.max_deg, [c.proof] * b, [c.cm] * b, [c.pos] * b, [c.evals] * b) == [0] * b
        counts.append(ctx.launches - before)
    assert counts[0] == counts[1] and counts[0] > 0


def test_errors_and_memory(ctx):
    c = Case(o.BLAKE3, 1, 4, 7, log_n=9)
    args = (c.h, 1, 4, 7, c.blowup, c.max_deg)
    live0 = ctx.mem_stats()[:2]
    assert ctx.fri_verify_batch(*args, [c.proof], [c.cm], [c.pos], [c.evals]) == [F.FRI_VERIFY_ACCEPT]
    assert ctx.mem_stats()[:2] == live0
    ev = c.evals.copy()
    ev[0, 0] ^= 1
    assert ctx.fri_verify_batch(*args, [c.proof, c.proof[:-2]], [c.cm, c.cm], [c.pos] * 2, [ev, c.evals]) == \
        [V(F.FRI_VERIFY_INVALID_LAYER_FOLDING, 0), F.FRI_VERIFY_MALFORMED]
    assert ctx.mem_stats()[:2] == live0
    bad_ev = c.evals.copy()
    bad_ev[2, 0] = o.P
    bad_pos = c.pos.copy()
    bad_pos[1] = c.N
    for kw, msg in [(dict(evaluations=[c.evals, bad_ev]), "proof 1"), (dict(positions=[c.pos, bad_pos]), "proof 1"),
                    (dict(commitments=[c.cm, c.cm[:-1]]), "proof 1")]:
        a = dict(proofs=[c.proof] * 2, commitments=[c.cm] * 2, positions=[c.pos] * 2, evaluations=[c.evals] * 2)
        a.update(kw)
        with pytest.raises(wf.WfError, match=msg):
            ctx.fri_verify_batch(*args, **a)
        assert ctx.mem_stats()[:2] == live0
    with pytest.raises(wf.WfError, match="error -3:.*folding factor 3"):
        ctx.fri_verify_batch(c.h, 1, 3, 7, c.blowup, c.max_deg, [c.proof], [c.cm], [c.pos], [c.evals])
    with pytest.raises(wf.WfError, match="error -3:.*unknown hash"):
        ctx.fri_verify_batch(9, 1, 4, 7, c.blowup, c.max_deg, [c.proof], [c.cm], [c.pos], [c.evals])
    assert ctx.mem_stats()[:2] == live0
