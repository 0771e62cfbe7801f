// air_host.hpp — the host-side form of an AIR description, shared by the prover (prover.cu), the trace checks
// (validate.cu) and the verifier (verify.cu).
#pragma once
#include "internal.hpp"
#include "constraints_generic.cuh"  // GEN_MAX_REGS / AUX_MAX_REGS: the register limits a description is parsed against

// Host-side AIR description (mirrors oracle/wf_prover.cpp `Air`; flat format documented at
// wf_prove_air in include/winterfell_b200.h)
// stride 0: Assertion::single; one value + stride: ::periodic; n / stride values: ::sequence
// (air/src/air/assertions/mod.rs:62-120). Main values: one word each; aux values: three words each.
struct AirAssertion { u64 column, first_step, stride; std::vector<u64> values; };
typedef AirAssertion AuxAssertion;
struct AirHost {
    u32 w = 0;
    // auxiliary segment (air/src/air/trace_info.rs:24-40): aw columns over E, nr random elements
    u32 aw = 0, nr = 0, aux_num_regs = 0;
    std::vector<std::pair<u32, std::vector<u32>>> aux_degrees;
    std::vector<u32> aux_prog;
    std::vector<AuxAssertion> aux_asserts;
    std::vector<std::pair<u32, std::vector<u32>>> all_degrees() const {  // context.rs:268-271
        auto r = degrees; r.insert(r.end(), aux_degrees.begin(), aux_degrees.end()); return r;
    }
    size_t num_constraints() const {  // transition then boundary constraints, main and aux (context.rs:205-207, :223-225)
        return degrees.size() + aux_degrees.size() + asserts.size() + aux_asserts.size();
    }
    std::vector<u64> pub_inputs;
    std::vector<std::pair<u32, std::vector<u32>>> degrees;
    std::vector<std::vector<u64>> periodic;
    std::vector<u64> consts;
    std::vector<u32> prog;  // 4 words per instruction
    u32 num_regs = 0;
    std::vector<AirAssertion> asserts;
    u32 exemptions = 1;
    bool is_fib = false;  // FibSmall x k: use the specialised kernel
    u32 fib_k = 0;
    std::vector<u64> fib_results;
    u32 log_ce_blowup() const {  // air/src/air/context.rs:87-100, transition/degree.rs min_blowup_factor
        u32 r = 1;
        for (auto& dg : all_degrees()) r = std::max(r, log2_ceil(dg.first + dg.second.size() - 1));
        return r;
    }
    u32 num_comp_cols(size_t n) const {  // context.rs:265-285
        size_t hi = 0;
        for (auto& dg : all_degrees()) {
            size_t e = (size_t)dg.first * (n - 1);
            for (u32 cyc : dg.second) e += (n / cyc) * (cyc - 1);
            hi = std::max(hi, e);
        }
        size_t div = n - exemptions;
        return (u32)std::max((hi - div + n - 1) / n, (size_t)1);
    }
    std::vector<AuxAssertion> sorted_aux_assertions() const {
        std::vector<AuxAssertion> a = aux_asserts;
        std::stable_sort(a.begin(), a.end(), [](const AuxAssertion& x, const AuxAssertion& y) {
            if (x.stride != y.stride) return x.stride < y.stride;
            if (x.first_step != y.first_step) return x.first_step < y.first_step;
            return x.column < y.column;
        });
        return a;
    }
    // periodic value tables (evaluator/periodic_table.rs:24-76): column j's polynomial (get_periodic_column_polys, air/mod.rs:325-360)
    // over offset^(n/L) <w_(L*ceb)>, concatenated; off / len: start and length of each table
    void periodic_ce_tables(size_t n, u32 log_ceb, std::vector<u64>& tab, std::vector<u32>& off, std::vector<u32>& len) const {
        for (auto& col : periodic) {
            const size_t L = col.size(), M = L << log_ceb;
            std::vector<u64> v = col;
            wf_host_dft(v, L, 1, true, 1);
            v.resize(M, 0);
            wf_host_dft(v, M, 1, false, gl_pow(GL_GENERATOR, n / L));
            off.push_back((u32)tab.size()); len.push_back((u32)M);
            tab.insert(tab.end(), v.begin(), v.end());
        }
    }
    std::vector<AirAssertion> sorted_assertions() const {  // assertions/mod.rs:301-315
        std::vector<AirAssertion> a = asserts;
        std::stable_sort(a.begin(), a.end(), [](const AirAssertion& x, const AirAssertion& y) {
            if (x.stride != y.stride) return x.stride < y.stride;
            if (x.first_step != y.first_step) return x.first_step < y.first_step;
            return x.column < y.column;
        });
        return a;
    }
};

// ---- AIR descriptions and proof options, as the prover (prover.cu) and the verifier (verify.cu) read them ----
struct Options {
    u32 num_queries, blowup, grinding, ext, folding, rem_max_deg, batch_c, batch_d, num_partitions, hash_rate;
    int hash_id;
    // PartitionOptions::partition_size::<E>(num_columns) (air/src/options.rs:428-438) in BASE columns, for `cols` columns of
    // extension degree `deg`; cols * deg = the row is hashed whole (RowMatrix::commit_to_rows, row_matrix.rs:191-193)
    u32 part_words(u32 cols, u32 deg) const {
        if (num_partitions <= 1) return cols * deg;
        const u32 min_ps = hash_rate / deg, ps = (cols + num_partitions - 1) / num_partitions;
        return (ps > min_ps ? ps : min_ps) * deg;
    }
};

static inline bool parse_air_host(const u64* d, size_t len, AirHost& a) {
    size_t p = 0;
    auto rd = [&](u64& v) { if (p >= len) return false; v = d[p++]; return true; };
    u64 v, cnt;
    if (!rd(v) || v == 0 || v > 255) return false;
    a.w = (u32)v;
    if (!rd(cnt) || cnt == 0 || cnt > 4096) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 base, nc;
        if (!rd(base) || !rd(nc) || base == 0 || nc > 16) return false;
        std::vector<u32> cyc;
        // TransitionConstraintDegree::with_cycles asserts cycle lengths that are powers of two >= 2 (transition/degree.rs:62-79)
        for (u64 j = 0; j < nc; j++) { if (!rd(v) || v < 2 || (v & (v - 1)) || v > (1ull << 32)) return false; cyc.push_back((u32)v); }
        if (base + nc - 1 > 128) return false;  // min_blowup_factor would exceed the largest blowup (options.rs:132-190)
        a.degrees.push_back({(u32)base, cyc});
    }
    if (!rd(cnt) || cnt > 64) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 ln;
        if (!rd(ln) || ln < 2 || (ln & (ln - 1))) return false;
        std::vector<u64> col;
        for (u64 j = 0; j < ln; j++) { if (!rd(v) || v >= GL_P) return false; col.push_back(v); }
        a.periodic.push_back(col);
    }
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) { if (!rd(v) || v >= GL_P) return false; a.consts.push_back(v); }
    if (!rd(v) || v > GEN_MAX_REGS || v < 2 * a.w + a.periodic.size()) return false;
    a.num_regs = (u32)v;
    if (!rd(cnt) || cnt > (1u << 20)) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 op, ds, x, y;
        if (!rd(op) || !rd(ds) || !rd(x) || !rd(y) || op > 4) return false;
        const u64 first_tmp = 2 * a.w + a.periodic.size();  // inputs are read-only: boundary terms re-read them
        if (op == 4) { if (ds >= a.degrees.size() || x >= a.num_regs) return false; }
        else if (op == 3) { if (ds >= a.num_regs || ds < first_tmp || x >= a.consts.size()) return false; }
        else if (ds >= a.num_regs || ds < first_tmp || x >= a.num_regs || y >= a.num_regs) return false;
        a.prog.insert(a.prog.end(), {(u32)op, (u32)ds, (u32)x, (u32)y});
    }
    if (!rd(cnt) || cnt == 0) return false;
    for (u64 i = 0; i < cnt; i++) {
        AirAssertion as;
        u64 nv;
        if (!rd(as.column) || !rd(as.first_step) || !rd(as.stride) || !rd(nv) || as.column >= a.w || nv == 0 || nv > len) return false;
        for (u64 j = 0; j < nv; j++) { if (!rd(v) || v >= GL_P) return false; as.values.push_back(v); }
        a.asserts.push_back(as);
    }
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) { if (!rd(v) || v >= GL_P) return false; a.pub_inputs.push_back(v); }
    if (!rd(v) || v == 0 || v > 8) return false;
    a.exemptions = (u32)v;
    if (p == len) return true;
    // optional aux section: [aw, nr, nTa, {base, ncyc, cyc...}*, aux_num_regs, nIa, {op,dst,a,b}*,
    //                        nAa, {column, first_step, stride, nvals, {v0, v1, v2} x nvals}*]
    if (!rd(v) || v == 0 || v > 255) return false;
    a.aw = (u32)v;
    if (!rd(v) || v > 255) return false;
    a.nr = (u32)v;
    if (!rd(cnt) || cnt == 0 || cnt > 4096) return false;   // context.rs:104-113
    for (u64 i = 0; i < cnt; i++) {
        u64 base, nc;
        if (!rd(base) || !rd(nc) || base == 0 || nc > 16) return false;
        std::vector<u32> cyc;
        for (u64 j = 0; j < nc; j++) { if (!rd(v) || v < 2 || (v & (v - 1)) || v > (1ull << 32)) return false; cyc.push_back((u32)v); }
        if (base + nc - 1 > 128) return false;
        a.aux_degrees.push_back({(u32)base, cyc});
    }
    const u64 first_tmp = 2 * a.w + 2 * a.aw + a.periodic.size() + a.nr;
    if (!rd(v) || v > AUX_MAX_REGS || v < first_tmp) return false;
    a.aux_num_regs = (u32)v;
    if (!rd(cnt) || cnt > (1u << 20)) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 op, ds, x, y;
        if (!rd(op) || !rd(ds) || !rd(x) || !rd(y) || op > 4) return false;
        if (op == 4) { if (ds >= a.aux_degrees.size() || x >= a.aux_num_regs) return false; }
        else if (op == 3) { if (ds >= a.aux_num_regs || ds < first_tmp || x >= a.consts.size()) return false; }
        else if (ds >= a.aux_num_regs || ds < first_tmp || x >= a.aux_num_regs || y >= a.aux_num_regs) return false;
        a.aux_prog.insert(a.aux_prog.end(), {(u32)op, (u32)ds, (u32)x, (u32)y});
    }
    if (!rd(cnt) || cnt == 0) return false;
    for (u64 i = 0; i < cnt; i++) {
        AuxAssertion as;
        u64 nv;
        if (!rd(as.column) || !rd(as.first_step) || !rd(as.stride) || !rd(nv) || as.column >= a.aw || nv == 0 || nv > len) return false;
        for (u64 j = 0; j < 3 * nv; j++) { if (!rd(v) || v >= GL_P) return false; as.values.push_back(v); }
        a.aux_asserts.push_back(as);
    }
    return p == len;
}

// cycle lengths of a TransitionConstraintDegree must not exceed the trace length (get_evaluation_degree,
// air/src/air/transition/degree.rs:85-97, divides trace_length by each cycle)
static inline int validate_degrees(wf_ctx* ctx, const std::vector<std::pair<u32, std::vector<u32>>>& degs, size_t n) {
    for (auto& dg : degs)
        for (u32 cyc : dg.second)
            if (cyc < 2 || (cyc & (cyc - 1)) || cyc > n) return wf_fail(ctx, WF_ERR_INVALID, "constraint degree cycle %u does not fit a trace of %zu rows", cyc, n);
    return WF_OK;
}

// Assertion validity (air/src/air/assertions/mod.rs:62-120, :166-230 validate_*)
static inline int validate_assertions(wf_ctx* ctx, const std::vector<AirAssertion>& as, size_t n, size_t words_per_value, const char* what) {
    for (auto& a : as) {
        const size_t nv = a.values.size() / words_per_value;
        bool ok = a.first_step < n && nv >= 1;
        if (a.stride != 0) ok = ok && a.stride >= 2 && !(a.stride & (a.stride - 1)) && a.stride <= n && a.first_step < a.stride;
        if (nv > 1) ok = ok && a.stride != 0 && !(nv & (nv - 1)) && nv * a.stride == n;   // sequence: one value per asserted step
        if (!ok) return wf_fail(ctx, WF_ERR_INVALID, "invalid %s", what);
    }
    // no two assertions may cover the same cell (Assertion::overlaps_with, assertions/mod.rs:175-208;
    // prepare_assertions panics on it, boundary/mod.rs:205-210)
    auto overlaps = [](const AirAssertion& s, const AirAssertion& o) {
        if (s.column != o.column) return false;
        if (s.first_step == o.first_step) return true;
        if (s.stride == o.stride) return false;
        const AirAssertion& lo = s.first_step < o.first_step ? s : o;
        const AirAssertion& hi = s.first_step < o.first_step ? o : s;
        if (lo.stride == 0) return false;  // the earlier one is a single assertion
        if (hi.stride == 0 || lo.stride < hi.stride) return (hi.first_step - lo.first_step) % lo.stride == 0;
        return false;
    };
    for (size_t i = 0; i < as.size(); i++)
        for (size_t j = i + 1; j < as.size(); j++)
            if (overlaps(as[i], as[j])) return wf_fail(ctx, WF_ERR_INVALID, "%s %zu overlaps with %zu", what, j, i);
    return WF_OK;
}

// The checks wf_prove_air / wf_eval_constraints run on an AIR description before touching the device, without a device:
// structure of the description, degrees against the blowup factor, periodic columns, assertion validity and overlaps
// (the panics of Air::new / BoundaryConstraints::new / prepare_assertions in the reference, returned as a status).
static inline int air_check_host(wf_ctx* ctx, const AirHost& air, uint32_t log_n, uint32_t blowup) {
    const size_t n = (size_t)1 << log_n;
    if (air.log_ce_blowup() > log2_ceil(blowup)) return wf_fail(ctx, WF_ERR_INVALID, "blowup factor too small for the constraint degrees");
    for (auto& col : air.periodic) if (col.size() > n) return wf_fail(ctx, WF_ERR_INVALID, "periodic column longer than the trace");
    CKI(validate_degrees(ctx, air.all_degrees(), n));
    CKI(validate_assertions(ctx, air.aux_asserts, n, 3, "aux assertion"));
    return validate_assertions(ctx, air.asserts, n, 1, "assertion");
}

// What the descriptions of one batch must share: everything but the public inputs and the assertion values. Returns the first
// part that differs, nullptr when the two have the same structure.
static inline const char* air_structure_mismatch(const AirHost& a, const AirHost& b) {
    // reasons[0..4]: count, columns, steps, strides, value counts
    auto layout = [](const std::vector<AirAssertion>& x, const std::vector<AirAssertion>& y, const char* const* reasons) -> const char* {
        if (x.size() != y.size()) return reasons[0];
        for (size_t i = 0; i < x.size(); i++) {
            if (x[i].column != y[i].column) return reasons[1];
            if (x[i].first_step != y[i].first_step) return reasons[2];
            if (x[i].stride != y[i].stride) return reasons[3];
            if (x[i].values.size() != y[i].values.size()) return reasons[4];
        }
        return nullptr;
    };
    static const char* const main_r[] = {"number of assertions", "assertion columns", "assertion steps", "assertion strides",
                                         "assertion value counts"};
    static const char* const aux_r[] = {"number of aux assertions", "aux assertion columns", "aux assertion steps",
                                        "aux assertion strides", "aux assertion value counts"};
    if (a.w != b.w) return "trace width";
    if (a.degrees != b.degrees) return "transition constraint degrees";
    if (a.periodic != b.periodic) return "periodic columns";
    if (a.consts != b.consts) return "constants";
    if (a.num_regs != b.num_regs || a.prog != b.prog) return "transition program";
    if (const char* why = layout(a.asserts, b.asserts, main_r)) return why;
    if (a.exemptions != b.exemptions) return "transition exemptions";
    if ((a.aw == 0) != (b.aw == 0)) return "aux segment";
    if (a.aw != b.aw || a.nr != b.nr) return "aux width or random elements";
    if (a.aux_degrees != b.aux_degrees) return "aux transition constraint degrees";
    if (a.aux_num_regs != b.aux_num_regs || a.aux_prog != b.aux_prog) return "aux transition program";
    return layout(a.aux_asserts, b.aux_asserts, aux_r);
}

// ---- proof transcript and wire format: the rules the provers (prover.cu) and the verifier (verify.cu) must share ----
// ProofOptions from the nine option words of the C ABI: opts[8] = hash_id | num_partitions << 8 | hash_rate << 16
// (ProofOptions::with_partitions, air/src/options.rs:193-200); 0 in either field is the default PartitionOptions::new(1, 1)
static inline Options options_from_words(const uint32_t* opts) {
    Options o;
    o.num_queries = opts[0]; o.blowup = opts[1]; o.grinding = opts[2]; o.ext = opts[3]; o.folding = opts[4];
    o.rem_max_deg = opts[5]; o.batch_c = opts[6]; o.batch_d = opts[7]; o.hash_id = (int)(opts[8] & 0xff);
    o.num_partitions = (opts[8] >> 8) & 0xff; o.hash_rate = (opts[8] >> 16) & 0xff;
    if (o.num_partitions == 0) o.num_partitions = 1;
    if (o.hash_rate == 0) o.hash_rate = 1;
    return o;
}
// ProofOptions::new / with_partitions asserts (air/src/options.rs:132-190, :410-417). The extension degree is left to the
// caller: the verifier answers a bad one with WF_VERIFY_CONTEXT, after its other checks
static inline bool options_in_range(const Options& o) {
    auto pow2 = [](u64 v) { return v && !(v & (v - 1)); };
    return o.num_queries >= 1 && o.num_queries <= 255 && pow2(o.blowup) && o.blowup >= 2 && o.blowup <= 128 && o.grinding <= 32 &&
           pow2(o.folding) && o.folding >= 2 && o.folding <= 16 && o.rem_max_deg <= 255 && pow2((u64)o.rem_max_deg + 1) &&
           o.batch_c <= 2 && o.batch_d <= 2 && o.num_partitions >= 1 && o.num_partitions <= 16 && o.hash_rate >= 1;
}

// the public coin's seed: Context::to_elements (context.rs:119-136; TraceInfo::to_elements, trace_info.rs:209-238), then
// the public inputs (prover/src/channel.rs:57-82)
static inline std::vector<u64> context_seed(const AirHost& air, size_t n, const Options& o) {
    const u64 c = air.w, ti0 = air.aw ? (((((c << 8) | 1) << 8) | air.aw) << 8) | air.nr : c << 8;
    std::vector<u64> seed = {ti0, (u64)n, 1, 0xFFFFFFFFULL, (u64)air.num_constraints(),
                             ((u64)o.ext << 24) | ((u64)o.folding << 16) | ((u64)o.rem_max_deg << 8) | o.blowup, o.grinding, o.num_queries};
    seed.insert(seed.end(), air.pub_inputs.begin(), air.pub_inputs.end());
    return seed;
}
// Context::write_into (context.rs:142-151): TraceInfo, modulus, ProofOptions, then the number of constraints.
// parse_proof (verify.cu) reads it back.
static inline void write_context(ByteVec& w, const AirHost& air, u32 log_n, const Options& o) {
    w.u8_((u8)air.w); w.u8_((u8)air.aw); w.u8_((u8)air.nr); w.u8_((u8)log_n); w.u16_(0);
    w.u8_(8); w.u64_(GL_P);
    w.u8_((u8)o.num_queries); w.u8_((u8)o.blowup); w.u8_((u8)o.grinding); w.u8_((u8)o.ext); w.u8_((u8)o.folding);
    w.u8_((u8)o.rem_max_deg); w.u8_((u8)o.batch_c); w.u8_((u8)o.batch_d); w.u8_((u8)o.num_partitions); w.u8_((u8)o.hash_rate);
    w.usize(air.num_constraints());
}

template <int D>
static inline GlExt<D> draw_ext(PublicCoin& coin) {
    GlExt<D> r = ext_zero<D>();
    coin.draw(D, r.v);
    return r;
}
// air/src/air/coefficients.rs:201-218: Linear / Algebraic / Horner batching of the coefficients drawn from the coin
template <int D>
static inline std::vector<GlExt<D>> draw_coeffs(PublicCoin& coin, u32 method, size_t n) {
    std::vector<GlExt<D>> r;
    if (method == 0) { for (size_t i = 0; i < n; i++) r.push_back(draw_ext<D>(coin)); return r; }
    GlExt<D> a = draw_ext<D>(coin), x = ext_from_base<D>(1);
    for (size_t i = 0; i < n; i++) { r.push_back(x); x = ext_mul(x, a); }
    if (method == 2) std::reverse(r.begin(), r.end());
    return r;
}

// Columns over E from the evaluations of their base-component columns (col_ext per column, 1 or D):
// H_j = sum_q phi^q * (component column q of j)
template <int D>
static inline std::vector<GlExt<D>> ext_from_components(const std::vector<GlExt<D>>& evals, u32 col_ext = D) {
    std::vector<GlExt<D>> r(evals.size() / col_ext);
    for (size_t j = 0; j < r.size(); j++) {
        GlExt<D> acc = ext_zero<D>();
        for (u32 q = 0; q < col_ext; q++) {
            GlExt<D> basis = ext_zero<D>();
            basis.v[q] = 1;
            acc = ext_add(acc, ext_mul(basis, evals[j * col_ext + q]));
        }
        r[j] = acc;
    }
    return r;
}

// OodFrame (air/src/proof/ood_frame.rs:59-72, :95-108) of the trace and the quotient columns, written to ood_t / ood_q when
// given; returns merge_ood_evaluations (:335-349), the hash of cur (trace, quotient) then next (trace, quotient) that the coin
// is reseeded with (prover/src/channel.rs:109-112)
template <int D>
static inline Digest ood_frames(int hash_id, const std::vector<GlExt<D>>& t_cur, const std::vector<GlExt<D>>& t_nxt,
                                const std::vector<GlExt<D>>& q_cur, const std::vector<GlExt<D>>& q_nxt, ByteVec* ood_t = nullptr,
                                ByteVec* ood_q = nullptr) {
    auto put = [](ByteVec& w, const std::vector<GlExt<D>>& v) { for (auto& e : v) for (int q = 0; q < D; q++) w.u64_(e.v[q]); };
    if (ood_t) { ood_t->u8_(2); put(*ood_t, t_cur); put(*ood_t, t_nxt); }
    if (ood_q) { ood_q->u8_(2); put(*ood_q, q_cur); put(*ood_q, q_nxt); }
    ByteVec m;
    put(m, t_cur); put(m, q_cur); put(m, t_nxt); put(m, q_nxt);
    return hh_hash_elements(hash_id, (const u64*)m.v.data(), m.v.size() / 8);
}

// The aux assertion values of Air::get_aux_assertions(aux_rand_elements) (air/src/air/mod.rs:279) as a callback sees them:
// [value][D] words out of the [value][3] of AirHost::aux_asserts, times R = 2^64 mod p when `mont`
static inline std::vector<u64> get_aux_assertion_words(const AirHost& air, int D, bool mont) {
    std::vector<u64> vals;
    for (auto& a : air.aux_asserts)
        for (size_t i = 0; i < a.values.size() / 3; i++)
            for (int k = 0; k < D; k++) vals.push_back(mont ? gl_mul(a.values[i * 3 + k], 0xFFFFFFFFULL) : a.values[i * 3 + k]);
    return vals;
}
// ... and back. A Montgomery word goes through gl_from_mont; a canonical one must be < p, else false (values part written)
static inline bool set_aux_assertion_words(AirHost& air, const u64* vals, int D, bool mont) {
    size_t q = 0;
    for (auto& a : air.aux_asserts)
        for (size_t i = 0; i < a.values.size() / 3; i++, q++)
            for (int k = 0; k < 3; k++) {
                u64 v = k < D ? vals[q * D + k] : 0;
                if (mont) v = gl_from_mont(v);
                else if (v >= GL_P) return false;
                a.values[i * 3 + k] = v;
            }
    return true;
}

// validate.cu: Trace::validate (prover/src/trace/mod.rs:86-201) and ConstraintEvaluationTable::validate_transition_degrees
// (prover/src/constraints/evaluation_table.rs:181-230, 421-477) on the device. A violation is a result (kind != WF_VALID and
// the reference's panic message), not an error: both return WF_OK when the check ran.
struct TraceReport {
    u32 kind = WF_VALID, index = 0, column = 0;
    u64 step = 0;
    std::vector<u64> first_fail;         // per transition constraint (main, then aux): first failing step, ~0 = none
    std::vector<u64> expected, actual;   // per transition constraint: declared and actual degrees (filled by the degree check)
    std::string msg;
};
// main: n x w trace-domain evaluations; aux: n x aw*D (nullptr for a single-segment AIR); rnd: [nr][D] canonical
int wf_check_trace(wf_ctx* ctx, const AirHost& air, const wf_mat* main, const wf_mat* aux, const u64* rnd, u32 log_n, int D,
                   TraceReport& rep);
// lde / alde: LDEs of the trace (and aux) segment at blowup 2^log_b >= the constraint evaluation blowup. Sets the report only
// when it is still WF_VALID (the trace check comes first in the reference); always fills expected / actual.
int wf_check_degrees(wf_ctx* ctx, const AirHost& air, const wf_mat* lde, const wf_mat* alde, const u64* rnd, u32 log_n, u32 log_b,
                     int D, TraceReport& rep);

// The two checks split into what a device computes on its share of the work and one host verdict, so that the sharded prover
// combines every rank's raw results (element-wise minimum for the trace check, the column blocks for the degrees) and gives
// the one-GPU prover's report and message.
// Trace check, raw results: [0] / [1] = the smallest (assertion << 40 | cell) over the failing main / aux assertion cells,
// [2 + j] = the first failing step of transition constraint j (main, then aux); ~0 = none.
struct TraceCheckPart {
    SegMatrix amain{};          // main assertions on columns [acol0, acol0 + amain.cols) only: n trace-domain rows of those columns
    u32 acol0 = 0;
    const wf_mat* main = nullptr;   // transitions: main (and aux, which is also where the aux assertions are read) trace rows
    const wf_mat* aux = nullptr;
    SegMatrix aasrt{};          // the aux assertions' n trace rows when `aux` holds a row window (base NULL: aux's own rows)
    size_t s0 = 0, s1 = 0;      // the steps checked: [s0, s1)
    size_t row0 = 0, rows = 0;  // rows != 0: main / aux hold trace rows [row0, row0 + rows), then row (row0 + rows) mod n
};
int wf_check_trace_part(wf_ctx* ctx, const AirHost& air, const TraceCheckPart& part, const u64* rnd, u32 log_n, int D, std::vector<u64>& raw);
void wf_trace_verdict(const AirHost& air, bool aux, int D, const std::vector<u64>& raw, TraceReport& rep);
// Degree check: CE rows [row0, row0 + ce_rows) (ce_rows = 0: all, row0 = 0) of every transition constraint over its divisor into
// `out` (ce_rows x n_mtr + n_atr*D, zeroed here); lde / alde hold those rows' LDE rows and the blowup halo rows when windowed
// (GenEvalParams::row0). Then deg1[col] = 1 + the degree of column col of `cols` (interpolated, and freed: cols = nullptr).
int wf_transition_columns(wf_ctx* ctx, const AirHost& air, const wf_mat* lde, const wf_mat* alde, const u64* rnd, u32 log_n, u32 log_b,
                          int D, size_t row0, size_t ce_rows, const SegMatrix& out);
int wf_column_degrees(wf_ctx* ctx, wf_mat*& cols, std::vector<u64>& deg1);
void wf_degree_verdict(const AirHost& air, bool aux, int D, u32 log_n, const std::vector<u64>& deg1, TraceReport& rep);
