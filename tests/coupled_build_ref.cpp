// tests/coupled_build_ref.cpp — CPU restatement of the aux build semantics (include/winterfell_b200.h wf_aux_build) for every
// column kind, COUPLED_RECURRENCE groups included; the reference the device build of coupled recurrences is tested against.
// TEST INFRASTRUCTURE: compiled by tests/coupled_builds.py into a temporary directory, on top of the oracle's field arithmetic
// and AIR parser (oracle/wf_prover.cpp, included as one translation unit). For kinds 0-6 it is tests/rational_build_ref.cpp.
//
// Per column j in order, per row i: the program over E gives num_i (OUT 0), den_i (OUT 1, default 1) and, in a
// LINEAR_RECURRENCE or RATIONAL_RECURRENCE column, m_i (OUT 2), in a RATIONAL_RECURRENCE column c_i (OUT 3); inv(0) = 0;
// t_i = num_i * inv(den_i); POINTWISE a[i] = t_i; RUNNING_PRODUCT / RUNNING_SUM a[0] = init, a[i+1] = a[i] * t_i / a[i] + t_i;
// LINEAR_RECURRENCE a[0] = init, a[i+1] = m_i * a[i] + t_i; RATIONAL_RECURRENCE a[0] = init,
// a[i+1] = (m_i * a[i] + num_i) * inv(c_i * a[i] + den_i). A COUPLED_RECURRENCE column j and the k - 1 COUPLED_MEMBER columns
// after it are one group: the leader's program gives t_r (OUT r) and M[r][c] (OUT 4 + 4r + c), unwritten slots 0;
// a_r[0] = init of column j + r, a[i+1] = M_i a[i] + t_i over E^k; all one row after the other.
// Registers: main rows i and (i+1) mod n, aux rows i and (i+1) mod n (columns before the column or group), periodic values
// col[i mod len], random elements, temporaries.
#include "wf_prover.cpp"

// trace [w][n], rand [nr][d], out [aw][n][d]. Returns 0, or -2 for a description this restatement cannot run.
extern "C" int wfr_coupled_build(const uint64_t* desc, size_t desc_len, const uint64_t* build, size_t build_len, const uint64_t* trace,
                                 size_t n, int d, const uint64_t* rand, uint64_t* out) {
    Air air;
    if (!parse_air(desc, desc_len, air) || !air.aw || n < 2 || d < 1 || d > 3) return -2;
    const size_t w = air.w, aw = air.aw, np = air.periodic.size(), nr = air.nr;
    size_t p = 0;
    auto rd = [&](u64& v) { if (p >= build_len) return false; v = build[p++]; return true; };
    u64 v, nc;
    if (!rd(v) || v != aw || !rd(nc) || nc > build_len) return -2;
    std::vector<u64> consts;
    for (u64 i = 0; i < nc; i++) { if (!rd(v)) return -2; consts.push_back(v); }
    Field F{d};
    std::vector<EE> rnd(nr);
    for (size_t i = 0; i < nr; i++) { rnd[i] = F.zero(); for (int k = 0; k < d; k++) rnd[i].v[k] = rand[i * d + k]; }
    auto aux_at = [&](size_t j, size_t i) { EE e = F.zero(); for (int k = 0; k < d; k++) e.v[k] = out[(j * n + i) * d + k]; return e; };
    auto put = [&](size_t j, size_t i, const EE& e) { for (int k = 0; k < d; k++) out[(j * n + i) * d + k] = e.v[k]; };
    const size_t pb = 2 * w + 2 * aw;
    for (size_t j = 0; j < aw;) {
        u64 kind, nregs, ni;
        EE init = F.zero();
        if (!rd(kind) || (kind > 2 && kind != 4 && kind != 6 && kind != 8) || !rd(init.v[0]) || !rd(init.v[1]) || !rd(init.v[2]) ||
            !rd(nregs) || nregs < pb + np + nr || !rd(ni) || ni > build_len)
            return -2;
        const u64 max_out = kind == 8 ? 19 : kind == 6 ? 3 : kind == 4 ? 2 : 1;
        std::vector<Instr> prog;
        for (u64 k = 0; k < ni; k++) {
            u64 op, ds, a, b;
            if (!rd(op) || !rd(ds) || !rd(a) || !rd(b)) return -2;
            if (op > 4 || (op != 4 && ds >= nregs) || (op == 4 && ds > max_out) || (op == 3 ? a >= consts.size() : a >= nregs) ||
                (op < 3 && b >= nregs))
                return -2;
            prog.push_back({(u32)op, (u32)ds, (u32)a, (u32)b});
        }
        // a group: the members' inits follow the leader's program
        std::vector<EE> acc{init};
        if (kind == 8) {
            while (j + acc.size() < aw && p < build_len && build[p] == 9) {
                EE e = F.zero();
                u64 nreg9, ni9;
                p++;
                if (!rd(e.v[0]) || !rd(e.v[1]) || !rd(e.v[2]) || !rd(nreg9) || !rd(ni9) || nreg9 || ni9) return -2;
                acc.push_back(e);
            }
            if (acc.size() < 2 || acc.size() > 4) return -2;
        }
        const size_t k = acc.size();
        std::vector<EE> r(nregs, F.zero());
        for (size_t i = 0; i < n; i++) {
            const size_t nx = (i + 1) % n;
            for (size_t c = 0; c < w; c++) { r[c] = F.from_base(trace[c * n + i]); r[w + c] = F.from_base(trace[c * n + nx]); }
            for (size_t c = 0; c < j; c++) { r[2 * w + c] = aux_at(c, i); r[2 * w + aw + c] = aux_at(c, nx); }
            for (size_t c = 0; c < np; c++) r[pb + c] = F.from_base(air.periodic[c][i % air.periodic[c].size()]);
            for (size_t c = 0; c < nr; c++) r[pb + np + c] = rnd[c];
            EE num = F.zero(), den = F.one(), mlt = F.one(), dm = F.zero();
            std::vector<EE> slot(20, F.zero());   // a group's OUT slots: t_r at r, M[r][c] at 4 + 4r + c
            for (const Instr& in : prog) {
                switch (in.op) {
                    case OP_ADD: r[in.dst] = F.add(r[in.a], r[in.b]); break;
                    case OP_SUB: r[in.dst] = F.sub(r[in.a], r[in.b]); break;
                    case OP_MUL: r[in.dst] = F.mul(r[in.a], r[in.b]); break;
                    case OP_CONST: r[in.dst] = F.from_base(consts[in.a]); break;
                    case OP_OUT:
                        if (kind == 8) slot[in.dst] = r[in.a];
                        else (in.dst == 0 ? num : in.dst == 1 ? den : in.dst == 2 ? mlt : dm) = r[in.a];
                        break;
                }
            }
            if (kind == 0) {
                put(j, i, F.mul(num, F.inv(den)));
                continue;
            }
            if (kind == 8) {
                for (size_t q = 0; q < k; q++) put(j + q, i, acc[q]);
                std::vector<EE> nxt(k);
                for (size_t q = 0; q < k; q++) {
                    nxt[q] = slot[q];
                    for (size_t c = 0; c < k; c++) nxt[q] = F.add(nxt[q], F.mul(slot[4 + 4 * q + c], acc[c]));
                }
                acc = nxt;
                continue;
            }
            put(j, i, acc[0]);
            if (kind == 6) {
                acc[0] = F.mul(F.add(F.mul(mlt, acc[0]), num), F.inv(F.add(F.mul(dm, acc[0]), den)));
            } else {
                const EE t = F.mul(num, F.inv(den));
                acc[0] = kind == 1 ? F.mul(acc[0], t) : kind == 2 ? F.add(acc[0], t) : F.add(F.mul(mlt, acc[0]), t);
            }
        }
        j += k;
    }
    return p == build_len ? 0 : -2;
}
