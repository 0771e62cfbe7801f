"""The stages after the commitments on inputs at the edges of their arithmetic: the delayed-reduction accumulator
(wf_acc_ops_dev) word for word against the exact model (combine_model.py), the out-of-domain evaluation on coefficient columns
aimed at its accumulators' reduction classes, the DEEP composition in coefficient and evaluation form at structured points
(0, 1, roots of unity, base-field points of the extensions, components p - 1) and at every scan-tile count, the refusal of a
DEEP point on the LDE domain, and the FRI fold at every folding factor, extension degree and layer size down to one row per
fold, on mini-DFT butterfly edges. Every check compares with Python integers or the oracle."""
import random

import numpy as np
import pytest

import combine_model as M
import ntt_model as NM
import winterfell_b200 as wf

pytestmark = pytest.mark.gpu
P = M.P


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


def _free(ctx, *objs):
    for o in objs:
        if o is not None:
            o.free()
    assert ctx.mem_stats()[0] == 0


def _zg(z, log_n):
    g = NM.root(log_n)
    return [v * g % P for v in z]


# ---- the accumulator ----
@pytest.mark.parametrize("k", [1, 2, 5, 64, 255])
def test_accumulator_words_and_reduction(ctx, k):
    import torch
    rng = random.Random(100 + k)
    rows = [(xs, ys) for _, xs, ys in M.dot_rows(k, rng)]
    rows += [([2**64 - 1] * k, [2**64 - 1] * k), ([P - 1] * k, [P - 1] * k)]
    rows += [([rng.randrange(2**64) for _ in range(k)], [rng.randrange(2**64) for _ in range(k)]) for _ in range(64)]
    n = len(rows)
    tx, ty = _dev([v for xs, _ in rows for v in xs]), _dev([v for _, ys in rows for v in ys])
    out = torch.empty(n * 6, dtype=torch.int64, device="cuda")
    ctx.acc_ops_dev(tx.data_ptr(), ty.data_ptr(), k, n, out.data_ptr())
    ctx.sync()
    got = _host(out)
    for i, (xs, ys) in enumerate(rows):
        w = M.dot(xs, ys)
        assert got[6 * i:6 * i + 5] == w, (k, i, [hex(v) for v in got[6 * i:6 * i + 5]], [hex(v) for v in w])
        assert got[6 * i + 5] == M.acc_reduce(w) == sum(x * y for x, y in zip(xs, ys)) % P, (k, i)
    assert ctx.mem_stats()[0] == 0


# ---- out-of-domain evaluation ----
def _ood_columns(ncols, n, pts, rng):
    """ncols base coefficient columns of n rows; every 64-row thread group aimed at one reduce class of one point and component"""
    d = len(pts[0])
    cache = {}
    cols = NM._rand(np.random.default_rng(rng.randrange(2**32)), (ncols, n))
    groups = -(-n // 64)
    for j in range(ncols):
        for g in range(groups):
            if 256 <= g < groups - 256:     # long columns: the first and last chunk are aimed, the middle is random
                continue
            key = ((j + g) % 2, (j + g // 2) % d)
            if key not in cache:
                cache[key] = M.ood_thread_rows(M.ood_mults(pts[key[0]], key[1]), rng)
            rows = cache[key]
            c = rows[(g + 3 * j) % len(rows)][1]
            cols[j, 64 * g:min(n, 64 * g + 64)] = c[:min(64, n - 64 * g)]
    return cols


def _ood_want(oracle, cols, d, col_ext, z):
    vals = [[int(v) for v in oracle.eval_poly_at(c, np.array(z, dtype=np.uint64))] for c in cols]
    if col_ext == 1:
        return vals
    out = []
    for J in range(len(cols) // d):   # extension column J = sum_q u^q (base column J d + q)
        acc = [0] * d
        for q in range(d):
            acc = M.ext_add(acc, M.ext_mul([int(q == i) for i in range(d)], vals[J * d + q]))
        out.append(acc)
    return out


OOD_CASES = ([(3, 3, 9, n) for n in (7, 8, 64, 2047, 2048, 2049, 4096)] +
             [(d, 1 if ncols % d else d, ncols, 2048 + 64) for d, ncols in ((1, 1), (2, 3), (3, 8), (1, 9), (2, 17), (3, 64), (1, 65))] +
             [(1, 1, 3, 4096), (2, 2, 2, 4096), (2, 1, 1, 1 << 22)])


@pytest.mark.parametrize("d,col_ext,ncols,n", OOD_CASES)
def test_ood_evaluation_on_aimed_columns(ctx, oracle, d, col_ext, ncols, n):
    rng = random.Random(7 * n + ncols + d)
    pts = [z for _, z in M.structured_points(d)]
    pairs = list(zip(pts, pts[1:] + pts[:1]))
    if n > 1 << 16:
        pairs = pairs[1:3]
    for z0, z1 in pairs:
        cols = _ood_columns(ncols, n, (z0, z1), rng)
        m = ctx.mat_from_host_columns(cols)
        o0, o1 = ctx.evaluate_at(m, d, col_ext, np.array(z0, dtype=np.uint64), np.array(z1, dtype=np.uint64))
        _free(ctx, m)
        for z, o in ((z0, o0), (z1, o1)):
            assert [[int(v) for v in r] for r in o] == _ood_want(oracle, cols, d, col_ext, z), (z0, z1)


# ---- DEEP composition, coefficient form ----
def _deep_main(c, n, d, rng):
    """c main columns of n rows: the first and last 4096 rows aimed at the deep_sum classes (deep_rows), random in between"""
    rows = M.deep_rows(c, rng)
    main = NM._rand(np.random.default_rng(rng.randrange(2**32)), (c, n))
    for i in list(range(min(n, 4096))) + list(range(max(4096, n - 4096), n)):
        main[:, i] = rows[i % len(rows)][1]
    return main


def _np_S(main, dc_main, extra):
    """S row by row: sum_j dc_j T_j (extension coefficient times base value) + sum of the extension terms in `extra`"""
    n, d = main.shape[1], dc_main.shape[1]
    S = np.zeros((n, d), dtype=np.uint64)
    for j in range(main.shape[0]):
        for q in range(d):
            S[:, q] = NM.fadd(S[:, q], NM.fmul(main[j], np.uint64(dc_main[j, q])))
    for coef, vals in extra:   # vals: [n, d]
        S = np.stack([NM.fadd(S[:, q], t) for q, t in enumerate(M.np_ext_mul(vals, np.array([coef], dtype=np.uint64)).T)], axis=1)
    return S


@pytest.mark.parametrize("d,log_n", [(1, 3), (2, 3), (3, 3), (1, 11), (3, 11), (2, 12), (3, 12), (2, 19), (1, 20)])
def test_deep_coefficient_form_at_structured_points(ctx, oracle, d, log_n):
    n, c, log_b = 1 << log_n, 9, 1 if log_n > 12 else 2
    rng = random.Random(log_n * 10 + d)
    main = _deep_main(c, n, d, rng)
    cons = oracle.rand_elems((1, n * d), log_n + d)
    dc = np.concatenate([M.deep_coeffs(c, d, d - 1), oracle.rand_elems((1, d), 9)])
    S = _np_S(main, dc[:c], [(dc[c], cons[0].reshape(n, d))])
    pts = M.structured_points(d)
    if log_n > 12:   # 1 tile run p = 0 (z = 0), b_tile = 1, b_items = 1; the vectorised scan costs seconds per point here
        pts = pts[:4] if d == 1 else pts[2:4]
    mm = ctx.mat_from_host_columns(main)
    cm = ctx.mat_from_host_columns(cons, ext_degree=d)
    for label, z in pts:
        b = np.array(z, dtype=np.uint64)
        bg = np.array(_zg(z, log_n), dtype=np.uint64)
        if n <= 1 << 12:
            q = [M.host_syn_div(oracle, S, x, d) for x in (b, bg)]
        else:
            q = [M.np_syn_div(S, x) for x in (b, bg)]
        want_coef = np.stack([NM.fadd(q[0][:, k], q[1][:, k]) for k in range(d)], axis=1)
        want = oracle.lde_rows(want_coef.reshape(1, n * d), 1 << log_b, d)
        got = ctx.deep_compose_polys(d, mm, None, cm, log_b, b, dc)
        rows = got.to_rows()
        got.free()
        assert np.array_equal(rows, want), label
    _free(ctx, mm, cm)


# ---- DEEP composition, evaluation form ----
def _eval_want(row, x, dc, vals, Sz, Szg, z, zg):
    d = len(z)
    S = [0] * d
    for j, v in enumerate(vals):   # v: d words (base values are [v, 0, ...])
        S = M.ext_add(S, M.ext_mul([int(t) for t in dc[j]], v))
    xe = [x] + [0] * (d - 1)
    a = M.ext_mul(M.ext_sub(S, Sz), M.ext_inv(M.ext_sub(xe, z)))
    b = M.ext_mul(M.ext_sub(S, Szg), M.ext_inv(M.ext_sub(xe, zg)))
    return M.ext_add(a, b)


def _on_domain(z, log_N):
    return all(v == 0 for v in z[1:]) and pow(z[0] * pow(7, P - 2, P), 1 << log_N, P) == 1


@pytest.mark.parametrize("d,aw", [(1, 0), (1, 1), (2, 0), (2, 2), (3, 0), (3, 1)])
def test_deep_evaluation_form_on_aimed_rows(ctx, oracle, d, aw):
    log_N, log_n, c, kc = 12, 9, 64 if d == 1 else 9, 2
    N = 1 << log_N
    rng = random.Random(d * 10 + aw)
    main = _deep_main(c, N, d, rng)
    aux = oracle.rand_elems((aw, N * d), 3 + d) if aw else None
    cons = oracle.rand_elems((kc, N * d), 5 + d)
    dc = np.concatenate([M.deep_coeffs(c, d, d - 1), oracle.rand_elems((aw + kc, d), 7)])
    cur, nxt = oracle.rand_elems((c + aw + kc, d), 11), oracle.rand_elems((c + aw + kc, d), 13)
    Sz, Szg = [0] * d, [0] * d
    for j in range(c + aw + kc):
        Sz = M.ext_add(Sz, M.ext_mul([int(v) for v in dc[j]], [int(v) for v in cur[j]]))
        Szg = M.ext_add(Szg, M.ext_mul([int(v) for v in dc[j]], [int(v) for v in nxt[j]]))
    mm = ctx.mat_from_host_columns(main)
    am = ctx.mat_from_host_columns(aux, ext_degree=d) if aw else None
    cm = ctx.mat_from_host_columns(cons, ext_degree=d)
    stride = N // 8   # deep_div_kernel: N / 8 threads of rows tid + r * stride, r < 8
    sample = sorted(set(list(range(0, 40)) + list(range(stride - 8, stride)) + list(range(7 * stride, 7 * stride + 40)) +
                        list(range(N - 40, N)) + [rng.randrange(N) for _ in range(40)]))
    w = NM.root(log_N)
    for label, z in M.structured_points(d):
        zg = _zg(z, log_n)
        if _on_domain(z, log_N) or _on_domain(zg, log_N):
            continue
        out = ctx.deep_compose(d, mm, am, cm, log_n, np.array(z, dtype=np.uint64), dc, cur, nxt)
        rows = out.to_rows()
        out.free()
        for i in sample:
            vals = [[int(main[j, i])] + [0] * (d - 1) for j in range(c)]
            for m_ in ([aux] if aw else []) + [cons]:
                vals += [[int(v) for v in m_[j, i * d:(i + 1) * d]] for j in range(m_.shape[0])]
            want = _eval_want(i, 7 * pow(w, i, P) % P, dc, vals, Sz, Szg, z, zg)
            assert [int(v) for v in rows[i]] == want, (label, i)
    _free(ctx, mm, am, cm)


@pytest.mark.parametrize("d", [1, 2, 3])
def test_deep_forms_agree_on_real_ldes_at_structured_points(ctx, oracle, d):
    log_n, log_b, c = 9, 3, 5
    n = 1 << log_n
    main = ctx.mat_from_host_columns(oracle.rand_elems((c, n), 20 + d))
    cons = ctx.mat_from_host_columns(oracle.rand_elems((1, n * d), 21 + d), ext_degree=d)
    coeffs = oracle.rand_elems((c + 1, d), 22 + d)
    lm, lc = main.lde(log_b), cons.lde(log_b)
    for label, z in M.structured_points(d):
        zg = _zg(z, log_n)
        za, zga = np.array(z, dtype=np.uint64), np.array(zg, dtype=np.uint64)
        a0, b0 = ctx.evaluate_at(main, d, 1, za, zga)
        a1, b1 = ctx.evaluate_at(cons, d, d, za, zga)
        want = ctx.deep_compose(d, lm, None, lc, log_n, za, coeffs, np.concatenate([a0, a1]), np.concatenate([b0, b1]))
        got = ctx.deep_compose_polys(d, main, None, cons, log_b, za, coeffs)
        assert np.array_equal(got.to_rows(), want.to_rows()), label
        got.free(); want.free()
    _free(ctx, main, cons, lm, lc)


@pytest.mark.parametrize("d", [1, 3])
def test_deep_point_on_the_lde_domain_is_refused(ctx, oracle, d):
    log_n, log_b = 6, 2
    n, log_N = 1 << log_n, log_n + log_b
    N = 1 << log_N
    main_cols = oracle.rand_elems((3, n), 30 + d)
    cons_cols = oracle.rand_elems((1, n * d), 31 + d)
    main = ctx.mat_from_host_columns(main_cols)
    cons = ctx.mat_from_host_columns(cons_cols, ext_degree=d)
    lm, lc = main.lde(log_b), cons.lde(log_b)
    coeffs = oracle.rand_elems((4, d), 32 + d)
    ood = np.zeros((4, d), dtype=np.uint64)
    x5 = 7 * pow(NM.root(log_N), 5, P) % P
    g_inv = pow(NM.root(log_n), P - 2, P)
    live = ctx.mem_stats()[0]
    for z0 in (x5, x5 * g_inv % P):   # z on the domain, then z*g on it
        z = np.array([z0] + [0] * (d - 1), dtype=np.uint64)
        assert _on_domain([int(v) for v in z], log_N)
        with pytest.raises(wf.WfError, match="LDE domain"):
            ctx.deep_compose(d, lm, None, lc, log_n, z, coeffs, ood, ood)
        assert ctx.mem_stats()[0] == live
        # the coefficient form is exact there: the serial syn_div of S, extended
        S = _np_S(main_cols, coeffs[:3], [(coeffs[3], cons_cols[0].reshape(n, d))])
        q = [M.host_syn_div(oracle, S, x, d) for x in (z, np.array(_zg([int(v) for v in z], log_n), dtype=np.uint64))]
        want_coef = np.stack([NM.fadd(q[0][:, k], q[1][:, k]) for k in range(d)], axis=1)
        got = ctx.deep_compose_polys(d, main, None, cons, log_b, z, coeffs)
        assert np.array_equal(got.to_rows(), oracle.lde_rows(want_coef.reshape(1, n * d), 1 << log_b, d))
        got.free()
    _free(ctx, main, cons, lm, lc)


# ---- FRI fold ----
def _fold_layers(L, nf, d, rng_np):
    m = L // nf
    aimed = M.fold_inputs(min(L, nf * 256), nf, d, rng_np)
    if m > 256:   # aimed rows first, random rows after
        full = NM._rand(rng_np, (L, d))
        ma = 256
        for k in range(nf):
            full[k * m:k * m + ma] = aimed[k * ma:(k + 1) * ma]
        aimed = full
    alt = np.zeros((L, d), dtype=np.uint64)
    alt[1::2] = P - 1
    return [("aimed", aimed), ("random", NM._rand(rng_np, (L, d))), ("constant p - 1", np.full((L, d), P - 1, dtype=np.uint64)),
            ("constant 0", np.zeros((L, d), dtype=np.uint64)), ("alternating 0, p - 1", alt)]


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("nf", [2, 4, 8, 16])
def test_fri_fold_every_shape_on_edges(ctx, oracle, d, nf):
    import torch
    rng_np = np.random.default_rng(d * 100 + nf)
    alphas = [("0", [0] * d), ("1", [1] + [0] * (d - 1)), ("p - 1", [P - 1] + [0] * (d - 1)),
              ("random", [int(v) for v in NM._rand(rng_np, (d,))])]
    if d > 1:
        alphas += [("base field", [5] + [0] * (d - 1)), ("all components p - 1", [P - 1] * d)]
    L = nf
    while L <= 1 << 14:
        for label, ev in _fold_layers(L, nf, d, rng_np):
            flat = ev.reshape(-1)
            t_in = torch.from_numpy(flat.view(np.int64).copy()).cuda()
            t_out = torch.empty(L // nf * d, dtype=torch.int64, device="cuda")
            tr = oracle.transpose_slice(flat, nf, d)
            for alabel, alpha in alphas:
                a = np.array(alpha, dtype=np.uint64)
                ctx.fri_fold_dev(t_in.data_ptr(), L, d, nf, a, t_out.data_ptr())
                ctx.sync()
                want = oracle.apply_drp(tr, nf, 7, a, d)
                assert (t_out.cpu().numpy().view(np.uint64) == want).all(), (L, label, alabel)
        L *= 2
    assert ctx.mem_stats()[0] == 0
