// tests/rational_build_ref.cpp — CPU restatement of the aux build semantics (include/winterfell_b200.h wf_aux_build) for every
// column kind, RATIONAL_RECURRENCE included; the reference the device build of rational recurrences is tested against.
// TEST INFRASTRUCTURE: compiled by tests/rational_builds.py into a temporary directory, on top of the oracle's field arithmetic
// and AIR parser (oracle/wf_prover.cpp, included as one translation unit). For kinds 0-4 it is tests/linrec_build_ref.cpp.
//
// Per column j in order, per row i: the program over E gives num_i (OUT 0), den_i (OUT 1, default 1) and, in a
// LINEAR_RECURRENCE or RATIONAL_RECURRENCE column, m_i (OUT 2), in a RATIONAL_RECURRENCE column c_i (OUT 3); inv(0) = 0;
// t_i = num_i * inv(den_i); POINTWISE a[i] = t_i; RUNNING_PRODUCT / RUNNING_SUM a[0] = init, a[i+1] = a[i] * t_i / a[i] + t_i;
// LINEAR_RECURRENCE a[0] = init, a[i+1] = m_i * a[i] + t_i; RATIONAL_RECURRENCE a[0] = init,
// a[i+1] = (m_i * a[i] + num_i) * inv(c_i * a[i] + den_i), one row after the other.
// Registers: main rows i and (i+1) mod n, aux rows i and (i+1) mod n (columns already built), periodic values col[i mod len],
// random elements, temporaries.
#include "wf_prover.cpp"

// trace [w][n], rand [nr][d], out [aw][n][d]. Returns 0, or -2 for a description this restatement cannot run.
extern "C" int wfr_rational_build(const uint64_t* desc, size_t desc_len, const uint64_t* build, size_t build_len, const uint64_t* trace,
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
    const size_t pb = 2 * w + 2 * aw;
    for (size_t j = 0; j < aw; j++) {
        u64 kind, nregs, ni;
        EE init = F.zero();
        if (!rd(kind) || (kind > 2 && kind != 4 && kind != 6) || !rd(init.v[0]) || !rd(init.v[1]) || !rd(init.v[2]) || !rd(nregs) ||
            nregs < pb + np + nr || !rd(ni) || ni > build_len)
            return -2;
        const u64 max_out = kind == 6 ? 3 : kind == 4 ? 2 : 1;
        std::vector<Instr> prog;
        for (u64 k = 0; k < ni; k++) {
            u64 op, ds, a, b;
            if (!rd(op) || !rd(ds) || !rd(a) || !rd(b)) return -2;
            if (op > 4 || (op != 4 && ds >= nregs) || (op == 4 && ds > max_out) || (op == 3 ? a >= consts.size() : a >= nregs) ||
                (op < 3 && b >= nregs))
                return -2;
            prog.push_back({(u32)op, (u32)ds, (u32)a, (u32)b});
        }
        std::vector<EE> r(nregs, F.zero());
        EE acc = init;
        for (size_t i = 0; i < n; i++) {
            const size_t nx = (i + 1) % n;
            for (size_t c = 0; c < w; c++) { r[c] = F.from_base(trace[c * n + i]); r[w + c] = F.from_base(trace[c * n + nx]); }
            for (size_t c = 0; c < j; c++) { r[2 * w + c] = aux_at(c, i); r[2 * w + aw + c] = aux_at(c, nx); }
            for (size_t c = 0; c < np; c++) r[pb + c] = F.from_base(air.periodic[c][i % air.periodic[c].size()]);
            for (size_t c = 0; c < nr; c++) r[pb + np + c] = rnd[c];
            EE num = F.zero(), den = F.one(), mlt = F.one(), dm = F.zero();
            for (const Instr& in : prog) {
                switch (in.op) {
                    case OP_ADD: r[in.dst] = F.add(r[in.a], r[in.b]); break;
                    case OP_SUB: r[in.dst] = F.sub(r[in.a], r[in.b]); break;
                    case OP_MUL: r[in.dst] = F.mul(r[in.a], r[in.b]); break;
                    case OP_CONST: r[in.dst] = F.from_base(consts[in.a]); break;
                    case OP_OUT: (in.dst == 0 ? num : in.dst == 1 ? den : in.dst == 2 ? mlt : dm) = r[in.a]; break;
                }
            }
            if (kind == 0) {
                const EE t = F.mul(num, F.inv(den));
                for (int k = 0; k < d; k++) out[(j * n + i) * d + k] = t.v[k];
                continue;
            }
            for (int k = 0; k < d; k++) out[(j * n + i) * d + k] = acc.v[k];
            if (kind == 6) {
                acc = F.mul(F.add(F.mul(mlt, acc), num), F.inv(F.add(F.mul(dm, acc), den)));
            } else {
                const EE t = F.mul(num, F.inv(den));
                acc = kind == 1 ? F.mul(acc, t) : kind == 2 ? F.add(acc, t) : F.add(F.mul(mlt, acc), t);
            }
        }
    }
    return p == build_len ? 0 : -2;
}
