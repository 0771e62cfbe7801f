// oracle/wf_prover.cpp — CPU restatement of winterfell's Prover::generate_proof and verifier::verify
// for the benchmark AIRs (TEST INFRASTRUCTURE; see wf_oracle.h). Follows prover/src/lib.rs:282-492,
// prover/src/channel.rs, prover/src/constraints/**, prover/src/composer/mod.rs, fri/src/prover/mod.rs,
// air/src/proof/*.rs (wire format) and verifier/src/{lib,channel,evaluator,composer}.rs +
// fri/src/verifier/mod.rs. PARITY UNPINNED at the proof level: the reference holds no golden proof bytes
// (SURVEY.md §8c) and cannot be built here (Rust, no cargo), so "byte-identical" is established as identical
// to this restatement + accepted by the restated verifier; the building blocks (field, NTT, LDE, hashes,
// Merkle, folding, coin) are pinned by the reference's own vectors in tests/test_oracle_kats.py, and this
// file's own output is pinned by tests/golden/proof_digests.json.
//
// AIR family "FibSmall x k": k independent copies of examples/src/fibonacci/fib_small/air.rs:16-69
// side by side (trace width 2k). k = 1 with start (1, 1) IS the reference's fib_small example
// (BASELINE configs[0]); k = 4 / 32 are the synthetic 8- / 64-column AIRs of configs[1] / [2]
// (SURVEY.md §8d). Pair j starts at (j+1, j+1); public inputs = the k results (for k = 1 exactly
// fib_small's single BaseElement).
#include <array>
#include <stdio.h>
#include <stdlib.h>

#include "wf_oracle.cpp"

extern "C" size_t wfo_partition_size(size_t num_partitions, size_t hash_rate, size_t ext_degree, size_t num_columns);

namespace {

struct Opts {
    u32 num_queries, blowup, grinding, ext, folding, rem_max_deg, batch_c, batch_d, num_partitions, hash_rate;
    int hash_id;
    // PartitionOptions::partition_size::<E>(num_columns) in BASE elements (air/src/options.rs:428-438): `cols` columns of
    // extension degree `deg`; == cols * deg when the row is hashed whole
    size_t part_words(size_t cols, size_t deg) const { return wfo_partition_size(num_partitions, hash_rate, deg, cols) * deg; }
};

struct EE {  // extension element of degree <= 3
    u64 v[3];
};
struct Field {
    int d;
    EE zero() const { return EE{{0, 0, 0}}; }
    EE one() const { return EE{{1, 0, 0}}; }
    EE from_base(u64 b) const { return EE{{b, 0, 0}}; }
    EE add(const EE& a, const EE& b) const { EE r = zero(); e_add(d, a.v, b.v, r.v); return r; }
    EE sub(const EE& a, const EE& b) const { EE r = zero(); e_sub(d, a.v, b.v, r.v); return r; }
    EE mul(const EE& a, const EE& b) const { EE r = zero(); e_mul(d, a.v, b.v, r.v); return r; }
    EE mul_base(const EE& a, u64 b) const { EE r = zero(); e_mul_base(d, a.v, b, r.v); return r; }
    EE inv(const EE& a) const { EE r = zero(); e_inv(d, a.v, r.v); return r; }
    bool eq(const EE& a, const EE& b) const { for (int i = 0; i < d; i++) if (a.v[i] != b.v[i]) return false; return true; }
    EE exp(EE a, u64 e) const {
        EE r = one();
        while (e) { if (e & 1) r = mul(r, a); a = mul(a, a); e >>= 1; }
        return r;
    }
};

struct Writer {
    std::vector<u8> b;
    void u8_(u8 x) { b.push_back(x); }
    void u16_(uint16_t x) { for (int i = 0; i < 2; i++) b.push_back((u8)(x >> (8 * i))); }
    void u32_(u32 x) { for (int i = 0; i < 4; i++) b.push_back((u8)(x >> (8 * i))); }
    void u64_(u64 x) { for (int i = 0; i < 8; i++) b.push_back((u8)(x >> (8 * i))); }
    void bytes(const void* p, size_t n) { const u8* q = (const u8*)p; b.insert(b.end(), q, q + n); }
    void usize(u64 v) { write_vint64(b, v); }
    void elems(const Field& F, const EE* e, size_t n) { for (size_t i = 0; i < n; i++) for (int k = 0; k < F.d; k++) u64_(e[i].v[k]); }
};

// ---- AIR description -------------------------------------------------------------------------------
// A generic single-segment AIR (air/src/air/mod.rs:174 `Air`): transition constraints as a small
// straight-line program over the evaluation frame, so that the same description drives the oracle,
// the device evaluator and the verifier. FibSmall x k is one instance (fib_air()).
// air/src/air/assertions/mod.rs:41-50. stride 0: Assertion::single; stride > 0 with one value: ::periodic;
// stride > 0 with n / stride values: ::sequence. Main-segment values are base elements (v[0] only),
// aux-segment values are elements of E.
struct Assertion { size_t column, first_step, stride; std::vector<EE> values; };
typedef Assertion AuxAssertion;
static Assertion single_assertion(size_t column, size_t step, u64 value) { return Assertion{column, step, 0, {EE{{value, 0, 0}}}}; }
struct Instr { u32 op, dst, a, b; };  // ADD/SUB/MUL dst = r[a] op r[b]; CONST dst = consts[a]; OUT result[dst] = r[a]
enum { OP_ADD = 0, OP_SUB = 1, OP_MUL = 2, OP_CONST = 3, OP_OUT = 4 };
struct Air {
    size_t w = 0, n = 0;
    Opts o;
    std::vector<u64> pub_inputs;                                 // PublicInputs::to_elements
    std::vector<std::pair<u32, std::vector<u32>>> degrees;       // TransitionConstraintDegree: base, cycles
    std::vector<std::vector<u64>> periodic;                      // get_periodic_column_values
    std::vector<u64> consts;
    std::vector<Instr> prog;
    u32 num_regs = 0;                                            // r[0..w) current, r[w..2w) next, r[2w..2w+np) periodic, temps
    std::vector<Assertion> asserts;
    u32 exemptions = 1;                                          // AirContext::num_transition_exemptions
    // auxiliary trace segment (air/src/air/trace_info.rs:24-40; at most one, as in the reference):
    // aw columns over E built from nr random elements drawn after the main commitment. The aux
    // program's registers: [0,w) main cur, [w,2w) main next, [2w,2w+aw) aux cur, [2w+aw,2w+2aw) aux
    // next, then periodic values, then the nr random elements, then temporaries — all of type E.
    size_t aw = 0, nr = 0;
    std::vector<std::pair<u32, std::vector<u32>>> aux_degrees;
    std::vector<Instr> aux_prog;
    u32 aux_num_regs = 0;
    std::vector<AuxAssertion> aux_asserts;
    // Air::get_aux_assertions(&self, aux_rand_elements) (air/src/air/mod.rs:279): when set, the VALUES of the aux assertions
    // are recomputed from the drawn random elements (prover: after the main commitment; verifier: same point of the
    // transcript). rand = [nr][d] words, values = [sum of nvals][d] words in description order (in: the description's
    // placeholders, out: the values to assert). Returns 0 on success.
    int (*aux_values_fn)(void*, const u64*, u64*) = nullptr;
    void* aux_values_user = nullptr;
    size_t width() const { return w; }
    size_t num_main_transition() const { return degrees.size(); }
    size_t num_transition() const { return degrees.size() + aux_degrees.size(); }  // context.rs:205-207
    size_t num_assertions() const { return asserts.size() + aux_asserts.size(); }  // context.rs:223-225
    std::vector<std::pair<u32, std::vector<u32>>> all_degrees() const {            // context.rs:268-271
        auto r = degrees; r.insert(r.end(), aux_degrees.begin(), aux_degrees.end()); return r;
    }
    size_t lde_size() const { return n * o.blowup; }
    size_t ce_blowup() const {  // air/src/air/context.rs:87-100 + transition/degree.rs min_blowup_factor
        size_t r = 0;
        for (auto& dg : all_degrees()) {
            size_t bound = dg.first + dg.second.size() - 1, p2 = 1;
            while (p2 < bound) p2 <<= 1;
            r = std::max(r, std::max(p2, (size_t)2));
        }
        return r;
    }
    size_t num_comp_cols() const {  // context.rs:265-285
        size_t hi = 0;
        for (auto& dg : all_degrees()) {
            size_t e = dg.first * (n - 1);  // degree.rs get_evaluation_degree
            for (u32 cyc : dg.second) e += (n / cyc) * (cyc - 1);
            hi = std::max(hi, e);
        }
        size_t div = n - exemptions;
        return std::max((hi - div + n - 1) / n, (size_t)1);
    }
    // Air::evaluate_transition through the program, over any field type T
    template <class T, class Sub, class Add, class Mul, class FromBase>
    void eval_transition(const T* cur, const T* nxt, const T* per, T* res, Sub sub, Add add, Mul mul, FromBase fb) const {
        std::vector<T> r(num_regs);
        for (size_t i = 0; i < w; i++) { r[i] = cur[i]; r[w + i] = nxt[i]; }
        for (size_t i = 0; i < periodic.size(); i++) r[2 * w + i] = per[i];
        for (const Instr& in : prog) {
            switch (in.op) {
                case OP_ADD: r[in.dst] = add(r[in.a], r[in.b]); break;
                case OP_SUB: r[in.dst] = sub(r[in.a], r[in.b]); break;
                case OP_MUL: r[in.dst] = mul(r[in.a], r[in.b]); break;
                case OP_CONST: r[in.dst] = fb(consts[in.a]); break;
                case OP_OUT: res[in.dst] = r[in.a]; break;
            }
        }
    }
    // Air::evaluate_aux_transition (air/src/air/mod.rs:248-260) through the aux program, over E
    template <class T, class Sub, class Add, class Mul, class FromBase>
    void eval_aux_transition(const T* mcur, const T* mnxt, const T* acur, const T* anxt, const T* per, const T* rnd, T* res,
                             Sub sub, Add add, Mul mul, FromBase fb) const {
        std::vector<T> r(aux_num_regs);
        for (size_t i = 0; i < w; i++) { r[i] = mcur[i]; r[w + i] = mnxt[i]; }
        for (size_t i = 0; i < aw; i++) { r[2 * w + i] = acur[i]; r[2 * w + aw + i] = anxt[i]; }
        const size_t pb = 2 * w + 2 * aw;
        for (size_t i = 0; i < periodic.size(); i++) r[pb + i] = per[i];
        for (size_t i = 0; i < nr; i++) r[pb + periodic.size() + i] = rnd[i];
        for (const Instr& in : aux_prog) {
            switch (in.op) {
                case OP_ADD: r[in.dst] = add(r[in.a], r[in.b]); break;
                case OP_SUB: r[in.dst] = sub(r[in.a], r[in.b]); break;
                case OP_MUL: r[in.dst] = mul(r[in.a], r[in.b]); break;
                case OP_CONST: r[in.dst] = fb(consts[in.a]); break;
                case OP_OUT: res[in.dst] = r[in.a]; break;
            }
        }
    }
    std::vector<AuxAssertion> aux_assertions() const {
        std::vector<AuxAssertion> a = aux_asserts;
        std::stable_sort(a.begin(), a.end(), [](const AuxAssertion& x, const AuxAssertion& y) {
            if (x.stride != y.stride) return x.stride < y.stride;
            if (x.first_step != y.first_step) return x.first_step < y.first_step;
            return x.column < y.column;
        });
        return a;
    }
    // assertions in the reference's sorted order (stride, first_step, column):
    // air/src/air/assertions/mod.rs:301-315, boundary/mod.rs prepare_assertions
    std::vector<Assertion> assertions() const {
        std::vector<Assertion> a = asserts;
        std::stable_sort(a.begin(), a.end(), [](const Assertion& x, const Assertion& y) {
            if (x.stride != y.stride) return x.stride < y.stride;
            if (x.first_step != y.first_step) return x.first_step < y.first_step;
            return x.column < y.column;
        });
        return a;
    }
    // periodic column polynomials (air/src/air/mod.rs:325-360): interpolation over the cycle
    std::vector<std::vector<u64>> periodic_polys() const {
        std::vector<std::vector<u64>> r;
        for (auto& col : periodic) {
            std::vector<u64> p = col;
            auto itw = get_inv_twiddles(p.size());
            interpolate_poly(p.data(), p.size(), 1, itw.data());
            r.push_back(p);
        }
        return r;
    }
};
typedef Air FibAir;  // the FibSmall x k entry points build an Air through fib_air()

// examples/src/fibonacci/fib_small/air.rs:16-69, k copies side by side: pair j starts at (j+1, j+1)
static Air fib_air(size_t k, size_t n, const u64* results, const Opts& o) {
    Air a;
    a.w = 2 * k; a.n = n; a.o = o;
    a.pub_inputs.assign(results, results + k);
    const u32 w = (u32)a.w;
    u32 t = 2 * w;  // first temp register
    for (u32 j = 0; j < k; j++) {
        a.degrees.push_back({1, {}});
        a.degrees.push_back({1, {}});
        // result[2j] = next[2j] - (cur[2j] + cur[2j+1]); result[2j+1] = next[2j+1] - (cur[2j+1] + next[2j])
        a.prog.push_back({OP_ADD, t, 2 * j, 2 * j + 1});
        a.prog.push_back({OP_SUB, t + 1, w + 2 * j, t});
        a.prog.push_back({OP_OUT, 2 * j, t + 1, 0});
        a.prog.push_back({OP_ADD, t, 2 * j + 1, w + 2 * j});
        a.prog.push_back({OP_SUB, t + 1, w + 2 * j + 1, t});
        a.prog.push_back({OP_OUT, 2 * j + 1, t + 1, 0});
        a.asserts.push_back(single_assertion(2 * j, 0, (u64)(j + 1)));
        a.asserts.push_back(single_assertion(2 * j + 1, 0, (u64)(j + 1)));
        a.asserts.push_back(single_assertion(2 * j + 1, n - 1, results ? results[j] : 0));
    }
    a.num_regs = t + 2;
    return a;
}

// flat u64 description shared with the product's C ABI (include/winterfell_b200.h wf_prove_air):
// [w, nT, {base, ncyc, cyc...}*, nP, {len, values...}*, nC, consts..., num_regs, nI, {op,dst,a,b}*,
//  nA, {column, first_step, stride, nvals, values...}*, nPub, pub..., exemptions]
static bool parse_air(const u64* d, size_t len, Air& a) {
    size_t p = 0;
    auto rd = [&](u64& v) { if (p >= len) return false; v = d[p++]; return true; };
    u64 v, cnt;
    if (!rd(v)) return false;
    a.w = v;
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 base, nc; if (!rd(base) || !rd(nc)) return false;
        std::vector<u32> cyc; for (u64 j = 0; j < nc; j++) { if (!rd(v)) return false; cyc.push_back((u32)v); }
        a.degrees.push_back({(u32)base, cyc});
    }
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 ln; if (!rd(ln)) return false;
        std::vector<u64> col; for (u64 j = 0; j < ln; j++) { if (!rd(v)) return false; col.push_back(v); }
        a.periodic.push_back(col);
    }
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) { if (!rd(v)) return false; a.consts.push_back(v); }
    if (!rd(v)) return false;
    a.num_regs = (u32)v;
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) { u64 op, ds, x, y; if (!rd(op) || !rd(ds) || !rd(x) || !rd(y)) return false; a.prog.push_back({(u32)op, (u32)ds, (u32)x, (u32)y}); }
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 c, fs, st, nv; if (!rd(c) || !rd(fs) || !rd(st) || !rd(nv) || nv == 0 || nv > len) return false;
        Assertion as{(size_t)c, (size_t)fs, (size_t)st, {}};
        for (u64 j = 0; j < nv; j++) { if (!rd(v)) return false; as.values.push_back(EE{{v, 0, 0}}); }
        a.asserts.push_back(as);
    }
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) { if (!rd(v)) return false; a.pub_inputs.push_back(v); }
    if (!rd(v)) return false;
    a.exemptions = (u32)v;
    if (p == len) return true;  // single-segment description
    // optional aux section: [aw, nr, nTa, {base, ncyc, cyc...}*, aux_num_regs, nIa, {op,dst,a,b}*,
    //                        nAa, {column, first_step, stride, nvals, {v0, v1, v2} x nvals}*]
    if (!rd(v)) return false;
    a.aw = v;
    if (!rd(v)) return false;
    a.nr = v;
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 base, nc; if (!rd(base) || !rd(nc)) return false;
        std::vector<u32> cyc; for (u64 j = 0; j < nc; j++) { if (!rd(v)) return false; cyc.push_back((u32)v); }
        a.aux_degrees.push_back({(u32)base, cyc});
    }
    if (!rd(v)) return false;
    a.aux_num_regs = (u32)v;
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) { u64 op, ds, x, y; if (!rd(op) || !rd(ds) || !rd(x) || !rd(y)) return false; a.aux_prog.push_back({(u32)op, (u32)ds, (u32)x, (u32)y}); }
    if (!rd(cnt)) return false;
    for (u64 i = 0; i < cnt; i++) {
        u64 c, fs, st, nv, v0, v1, v2; if (!rd(c) || !rd(fs) || !rd(st) || !rd(nv) || nv == 0 || nv > len) return false;
        Assertion as{(size_t)c, (size_t)fs, (size_t)st, {}};
        for (u64 j = 0; j < nv; j++) { if (!rd(v0) || !rd(v1) || !rd(v2)) return false; as.values.push_back(EE{{v0, v1, v2}}); }
        a.aux_asserts.push_back(as);
    }
    return p == len && a.aw > 0 && !a.aux_degrees.empty() && !a.aux_asserts.empty();  // context.rs:104-113
}

static std::vector<u64> context_elements(const FibAir& air) {
    // air/src/proof/context.rs:119-136; air/src/air/trace_info.rs:209-238; air/src/options.rs:294-305
    std::vector<u64> e;
    if (air.aw == 0) e.push_back(((u64)air.width() << 8) | 0);  // main width, 0 aux segments
    else e.push_back((((((u64)air.width() << 8) | 1) << 8 | air.aw) << 8) | air.nr);
    e.push_back((u64)air.n);
    e.push_back(1);                            // low half of the modulus bytes
    e.push_back(0xFFFFFFFFULL);                // high half
    e.push_back((u64)(air.num_assertions() + air.num_transition()));  // prover/src/channel.rs:58-59
    const Opts& o = air.o;
    e.push_back(((u64)o.ext << 24) | ((u64)o.folding << 16) | ((u64)o.rem_max_deg << 8) | o.blowup);
    e.push_back(o.grinding);
    e.push_back(o.num_queries);
    return e;
}
static void write_context(Writer& w, const FibAir& air) {
    // context.rs:142-151; trace_info.rs:240-264; options.rs:307-320
    w.u8_((u8)air.width()); w.u8_((u8)air.aw); w.u8_((u8)air.nr);
    w.u8_((u8)__builtin_ctzll(air.n));
    w.u16_(0);  // no trace meta
    w.u8_(8);
    w.u64_(P);
    const Opts& o = air.o;
    w.u8_((u8)o.num_queries); w.u8_((u8)o.blowup); w.u8_((u8)o.grinding); w.u8_((u8)o.ext);
    w.u8_((u8)o.folding); w.u8_((u8)o.rem_max_deg); w.u8_((u8)o.batch_c); w.u8_((u8)o.batch_d);
    w.u8_((u8)o.num_partitions); w.u8_((u8)o.hash_rate);
    w.usize(air.num_assertions() + air.num_transition());
}

struct Coin {
    wfo_coin c;
    Coin(int h, const std::vector<u64>& seed) { wfo_coin_new(&c, h, seed.data(), seed.size()); }
    void reseed(const u8* d) { wfo_coin_reseed(&c, d); }
    EE draw(const Field& F) { EE r = F.zero(); if (coin_draw(&c, F.d, r.v)) abort(); return r; }
    // air/src/air/coefficients.rs:201-218 (+ :84-94 reversal for Horner)
    std::vector<EE> draw_coeffs(const Field& F, int method, size_t n) {
        std::vector<EE> r;
        if (method == 0) { for (size_t i = 0; i < n; i++) r.push_back(draw(F)); return r; }
        EE alpha = draw(F), x = F.one();
        for (size_t i = 0; i < n; i++) { r.push_back(x); x = F.mul(x, alpha); }
        if (method == 2) std::reverse(r.begin(), r.end());
        return r;
    }
};

static EE horner_base(const Field& F, const u64* p, size_t n, const EE& x) {  // polynom::eval, base coefficients
    EE acc = F.zero();
    for (size_t i = n; i-- > 0;) { acc = F.mul(acc, x); acc.v[0] = f_add(acc.v[0], p[i]); }
    return acc;
}
static EE horner_ext(const Field& F, const EE* p, size_t n, const EE& x) {
    EE acc = F.zero();
    for (size_t i = n; i-- > 0;) acc = F.add(F.mul(acc, x), p[i]);
    return acc;
}

// ---- boundary constraint groups (air/src/air/boundary/mod.rs:154 group_constraints) -----------------
// BTreeMap keyed by (stride, first_step); divisor x^a - b with a = number of asserted steps and
// b = g^(a * first_step) (air/src/air/divisor.rs:44-56 from_assertion). A constraint's value polynomial
// (boundary/constraint.rs:47-75): one coefficient for single / periodic assertions; for sequence
// assertions the interpolant of the values over the size-a subgroup, evaluated at x * g^(-first_step).
struct BoundaryEntry { size_t col; std::vector<EE> poly; u64 x_offset; size_t first_step; EE cc; };
struct BoundaryGroup { u64 a, b; std::vector<BoundaryEntry> e; };
typedef BoundaryGroup AuxBoundaryGroup;
static std::vector<BoundaryGroup> group_constraints(const Air& air, const std::vector<Assertion>& as, const EE* bcoef, int d) {
    u64 g = root_of_unity((u32)__builtin_ctzll(air.n));
    std::map<std::pair<size_t, size_t>, BoundaryGroup> m;
    for (size_t i = 0; i < as.size(); i++) {
        auto key = std::make_pair(as[i].stride, as[i].first_step);
        auto it = m.find(key);
        if (it == m.end()) {
            BoundaryGroup G;
            G.a = as[i].stride == 0 ? 1 : air.n / as[i].stride;  // assertions/mod.rs:284-295 get_num_steps
            G.b = as[i].first_step == 0 ? 1 : f_exp(g, G.a * as[i].first_step);
            it = m.insert({key, G}).first;
        }
        BoundaryEntry e{as[i].column, as[i].values, 1, as[i].first_step, bcoef[i]};
        for (auto& v : e.poly) for (int k = d; k < 3; k++) v.v[k] = 0;
        if (e.poly.size() > 1) {  // boundary/constraint.rs:58-68
            const size_t L = e.poly.size();
            std::vector<u64> flat(L * d);
            for (size_t j = 0; j < L; j++) for (int k = 0; k < d; k++) flat[j * d + k] = e.poly[j].v[k];
            auto itw = get_inv_twiddles(L);
            interpolate_poly(flat.data(), L, d, itw.data());
            for (size_t j = 0; j < L; j++) for (int k = 0; k < d; k++) e.poly[j].v[k] = flat[j * d + k];
            if (as[i].first_step != 0) e.x_offset = f_exp(f_inv(g), as[i].first_step);
        }
        it->second.e.push_back(e);
    }
    std::vector<BoundaryGroup> r;
    for (auto& kv : m) r.push_back(kv.second);
    return r;
}
static std::vector<BoundaryGroup> boundary_groups(const Air& air, const std::vector<EE>& bcoef) {
    return group_constraints(air, air.assertions(), bcoef.data(), 1);
}
// constraints against the auxiliary segment (boundary/mod.rs:121-128): same grouping, values in E
static std::vector<BoundaryGroup> aux_boundary_groups(const Air& air, const EE* bcoef) {
    return group_constraints(air, air.aux_assertions(), bcoef, (int)air.o.ext);
}
// LargePolyConstraint::new (prover/src/constraints/evaluator/boundary.rs:400-425): the value polynomial
// evaluated over the whole CE domain (offset 7); row i of the CE domain reads entry (i - first_step *
// ce_blowup) mod ce (:428-445). SmallPolyConstraint (:340-375, Horner at x * x_offset) computes the same
// values, so one table serves both. Returned flat [ce][d]; empty for single-value constraints.
static std::vector<u64> sequence_table(const BoundaryEntry& e, int d, size_t ce) {
    const size_t L = e.poly.size();
    if (L <= 1) return {};
    std::vector<u64> flat(L * d), out(ce * d);
    for (size_t j = 0; j < L; j++) for (int k = 0; k < d; k++) flat[j * d + k] = e.poly[j].v[k];
    auto tw = get_twiddles(L);
    evaluate_poly_with_offset(flat.data(), L, d, tw.data(), GENERATOR, ce / L, out.data());
    return out;
}
// builds the auxiliary segment (Prover::build_aux_trace, prover/src/lib.rs:236-247): rand [nr][d] words,
// out [aw][n][d] words
typedef int (*AuxBuilder)(void* user, const u64* rand_elements, u64* aux_out);

// transition divisor exemption points g^(n-1), ..., g^(n-k) (divisor.rs:31-41 from_transition)
static std::vector<u64> exemption_points(const Air& air) {
    u64 g = root_of_unity((u32)__builtin_ctzll(air.n));
    std::vector<u64> r;
    for (size_t st = air.n - air.exemptions; st < air.n; st++) r.push_back(f_exp(g, st));
    return r;
}

// PeriodicValueTable::new (prover/src/constraints/evaluator/periodic_table.rs:24-76): column j evaluated
// over the coset offset^(n/L) <w_(L*ceb)>; row i of the CE domain reads entry i mod (L * ce_blowup)
static std::vector<std::vector<u64>> periodic_value_table(const Air& air) {
    std::vector<std::vector<u64>> ptab;
    for (auto& poly : air.periodic_polys()) {
        size_t L = poly.size();
        std::vector<u64> ev(L * air.ce_blowup());
        auto tw = get_twiddles(L);
        evaluate_poly_with_offset(poly.data(), L, 1, tw.data(), f_exp(GENERATOR, air.n / L), air.ce_blowup(), ev.data());
        ptab.push_back(ev);
    }
    return ptab;
}

// ---- constraint evaluation over the CE domain ----------------------------------------------------------
// DefaultConstraintEvaluator::evaluate (evaluator/default.rs:60-118) fused with ConstraintEvaluationTable::combine
// (evaluation_table.rs:163-407), one CE row at a time from that row's frames, in plain per-row formulas: x^a by f_exp,
// one f_inv per divisor, table rows by % size. The prover runs it over the whole domain; wfo_eval_constraint_rows over
// the rows a test names. ccoef: [main transition, aux transition | main assertions, aux assertions (sorted order)].
struct CeEvaluator {
    const Air& air;
    Field F;
    size_t n, ce, c, aw;
    u64 g_ce;
    std::vector<EE> tcoef, tcoef_aux;
    std::vector<BoundaryGroup> groups, aux_groups;
    std::vector<std::vector<std::vector<u64>>> gtab, agtab;
    std::vector<u64> exempt;
    std::vector<std::vector<u64>> ptab;
    const EE* rnd;
    struct Scratch {
        std::vector<u64> tev, per;
        std::vector<EE> mc, mn, ac, an, pe, aev;
    };
    CeEvaluator(const Air& a, int d, const std::vector<EE>& ccoef, const EE* rand_elems)
        : air(a), F{d}, n(a.n), ce(a.n * a.ce_blowup()), c(a.width()), aw(a.aw), rnd(rand_elems) {
        const size_t nTm = air.num_main_transition(), nT = air.num_transition();
        tcoef.assign(ccoef.begin(), ccoef.begin() + nTm);          // transition/mod.rs:63-72 split
        tcoef_aux.assign(ccoef.begin() + nTm, ccoef.begin() + nT);
        std::vector<EE> bcoef(ccoef.begin() + nT, ccoef.begin() + nT + air.asserts.size());  // boundary/mod.rs:108-110
        groups = boundary_groups(air, bcoef);
        aux_groups = aux_boundary_groups(air, ccoef.data() + nT + air.asserts.size());
        g_ce = root_of_unity((u32)__builtin_ctzll(ce));
        exempt = exemption_points(air);
        // periodic value table (evaluator/periodic_table.rs:24-76): column j evaluated over the coset
        // offset^(n/L) <w_(L*ceb)>, row i of the CE domain reads entry i mod (L*ceb)
        ptab = periodic_value_table(air);
        gtab.resize(groups.size());
        agtab.resize(aux_groups.size());
        for (size_t gi = 0; gi < groups.size(); gi++) for (auto& e : groups[gi].e) gtab[gi].push_back(sequence_table(e, 1, ce));
        for (size_t gi = 0; gi < aux_groups.size(); gi++) for (auto& e : aux_groups[gi].e) agtab[gi].push_back(sequence_table(e, d, ce));
    }
    Scratch scratch() const {
        Scratch s;
        s.tev.resize(tcoef.size()); s.per.resize(ptab.size());
        s.mc.resize(c); s.mn.resize(c); s.ac.resize(aw); s.an.resize(aw); s.pe.resize(ptab.size()); s.aev.resize(tcoef_aux.size());
        return s;
    }
    // CE row i from its frames: main rows cur / nxt [c], aux rows ar / arn [aw][d] (ignored without an aux segment)
    EE row(size_t i, const u64* cur, const u64* nxt, const u64* ar, const u64* arn, Scratch& s) const {
        const int d = F.d;
        auto e_sub = [&](const EE& x, const EE& y) { return F.sub(x, y); };
        auto e_add = [&](const EE& x, const EE& y) { return F.add(x, y); };
        auto e_mul = [&](const EE& x, const EE& y) { return F.mul(x, y); };
        auto e_fb = [&](u64 v) { return F.from_base(v); };
        for (size_t j = 0; j < ptab.size(); j++) s.per[j] = ptab[j][i % ptab[j].size()];
        std::fill(s.tev.begin(), s.tev.end(), 0);
        air.eval_transition(cur, nxt, s.per.data(), s.tev.data(), f_sub, f_add, f_mul, [](u64 v) { return v; });
        EE t = F.zero();
        for (size_t j = 0; j < s.tev.size(); j++) t = F.add(t, F.mul_base(tcoef[j], s.tev[j]));
        if (aw) {  // evaluator/default.rs:306-341 evaluate_aux_transition
            for (size_t j = 0; j < c; j++) { s.mc[j] = F.from_base(cur[j]); s.mn[j] = F.from_base(nxt[j]); }
            for (size_t j = 0; j < aw; j++) {
                s.ac[j] = F.zero(); s.an[j] = F.zero();
                for (int k = 0; k < d; k++) { s.ac[j].v[k] = ar[j * d + k]; s.an[j].v[k] = arn[j * d + k]; }
            }
            for (size_t j = 0; j < s.per.size(); j++) s.pe[j] = F.from_base(s.per[j]);
            std::fill(s.aev.begin(), s.aev.end(), F.zero());
            air.eval_aux_transition(s.mc.data(), s.mn.data(), s.ac.data(), s.an.data(), s.pe.data(), rnd, s.aev.data(), e_sub, e_add,
                                    e_mul, e_fb);
            for (size_t j = 0; j < s.aev.size(); j++) t = F.add(t, F.mul(s.aev[j], tcoef_aux[j]));
        }
        u64 x = f_mul(f_exp(g_ce, i), GENERATOR);                  // domain.rs get_ce_x_at
        u64 zt = f_inv(f_sub(f_exp(x, n), 1));                     // 1 / (x^n - 1)
        u64 ex = 1;
        for (u64 e : exempt) ex = f_mul(ex, f_sub(x, e));          // divisor.rs evaluate_exemptions_at
        EE acc = F.mul_base(t, f_mul(zt, ex));                     // evaluation_table.rs:343-366
        for (size_t gi = 0; gi < groups.size(); gi++) {
            auto& G = groups[gi];
            EE bsum = F.zero();
            for (size_t q = 0; q < G.e.size(); q++) {              // evaluator/boundary.rs Single / Small / LargePoly
                const BoundaryEntry& e = G.e[q];
                u64 val = e.poly.size() == 1 ? e.poly[0].v[0] : gtab[gi][q][(i + ce - (e.first_step * air.ce_blowup()) % ce) % ce];
                bsum = F.add(bsum, F.mul_base(e.cc, f_sub(cur[e.col], val)));
            }
            acc = F.add(acc, F.mul_base(bsum, f_inv(f_sub(f_exp(x, G.a), G.b))));  // :329-340
        }
        for (size_t gi = 0; gi < aux_groups.size(); gi++) {  // evaluator/boundary.rs:228-260 aux constraints
            auto& G = aux_groups[gi];
            EE bsum = F.zero();
            for (size_t q = 0; q < G.e.size(); q++) {
                const BoundaryEntry& e = G.e[q];
                EE val = e.poly[0];
                if (e.poly.size() > 1) {
                    size_t idx = (i + ce - (e.first_step * air.ce_blowup()) % ce) % ce;
                    val = F.zero();
                    for (int k = 0; k < d; k++) val.v[k] = agtab[gi][q][idx * d + k];
                }
                bsum = F.add(bsum, F.mul(F.sub(s.ac[e.col], val), e.cc));
            }
            acc = F.add(acc, F.mul_base(bsum, f_inv(f_sub(f_exp(x, G.a), G.b))));
        }
        return acc;
    }
};

// ---- the proof -----------------------------------------------------------------------------------
struct ProofParts {
    std::vector<u8> bytes;
};

// Byte range of a section of opened values in the proof (offset, length).
struct Section { size_t off = 0, len = 0; };

// returns where the opened values were written
static Section queries_for(const Field& F, int h, const u64* rows_mat, size_t row_words, const std::vector<u8>& leaves,
                           const std::vector<u8>& nodes, size_t N, const std::vector<u64>& pos, Writer& w) {
    (void)F;
    // air/src/proof/queries.rs:51-78,138-146 + trace_lde/default/mod.rs:284-297
    Writer vals;
    for (u64 p : pos) vals.bytes(rows_mat + p * row_words, row_words * 8);
    std::vector<u8> lv(pos.size() * 32), pr(64 + pos.size() * 40 * 33);
    long pl = merkle_prove_batch(leaves.data(), nodes.data(), N, pos.data(), pos.size(), lv.data(), pr.data(), pr.size(), digest_len(h));
    if (pl < 0) abort();
    (void)h;
    w.usize(vals.b.size());
    Section s{w.b.size(), vals.b.size()};
    w.bytes(vals.b.data(), vals.b.size());
    w.usize((u64)pl); w.bytes(pr.data(), (size_t)pl);
    return s;
}

// ---- dishonest proofs -----------------------------------------------------------------------------
// The oracle is test infrastructure, so it cheats on request: a proof whose every opening verifies and that is still wrong
// is the only kind that reaches the verifier's FRI folding and remainder checks. A tamper names a target, an index, a row
// (or every row) and a delta in E (d words, each < p; base-field targets use word 0):
//   T_MAIN_LDE / T_AUX_LDE / T_CONSTRAINT_LDE, column `index`: the committed and opened rows of that LDE carry the delta;
//     constraint evaluation, the OOD frame and the DEEP polynomial use the honest values.
//   T_FRI_LAYER, layer `index` (0 = the DEEP codeword, index = number of layers: the remainder's codeword), row = position in
//     the layer's domain: the delta is added before the layer is committed, and the next layer is folded from it.
//   T_REMAINDER: the delta is added to serialized remainder coefficient `index` before it is hashed into the transcript.
//   T_REMAINDER_LONG: `index` (>= 1) zero coefficients are put in front of the remainder (its highest degrees: the
//     polynomial keeps its values, only its length is wrong).
//   T_FLIP_TRACE / T_FLIP_AUX / T_FLIP_CONSTRAINT / T_FLIP_FRI (layer `index`): once the proof is written, bit
//     (delta[0] mod 8) of byte `row` (ALL_ROWS: byte 0) of that section's opened values is flipped.
enum { T_MAIN_LDE = 0, T_AUX_LDE, T_CONSTRAINT_LDE, T_FRI_LAYER, T_REMAINDER, T_REMAINDER_LONG,
       T_FLIP_TRACE, T_FLIP_AUX, T_FLIP_CONSTRAINT, T_FLIP_FRI };
constexpr u64 ALL_ROWS = ~(u64)0;
struct Tamper { u64 target, index, row, delta[3]; };
struct Tampers {
    std::vector<Tamper> list;
    std::vector<u64> positions;   // out: the query positions the proof opens
};

// the matrix [rows][cols * d] as committed: `m` itself, or a copy carrying the deltas of `target`
static const u64* committed(const Tampers* tp, int target, const std::vector<u64>& m, size_t rows, size_t cols, int d,
                            std::vector<u64>& copy) {
    if (!tp) return m.data();
    for (const Tamper& t : tp->list) {
        if ((int)t.target != target) continue;
        if (copy.empty()) copy = m;
        const size_t r0 = t.row == ALL_ROWS ? 0 : t.row, r1 = t.row == ALL_ROWS ? rows : t.row + 1;
        for (size_t r = r0; r < r1; r++)
            for (int k = 0; k < d; k++) copy[(r * cols + t.index) * d + k] = f_add(copy[(r * cols + t.index) * d + k], t.delta[k]);
    }
    return copy.empty() ? m.data() : copy.data();
}
// the deltas of FRI layer `layer` on its evaluations [len][d]
static void tamper_layer(const Tampers* tp, size_t layer, std::vector<u64>& ev, size_t len, int d) {
    if (!tp) return;
    for (const Tamper& t : tp->list) {
        if (t.target != T_FRI_LAYER || t.index != layer) continue;
        const size_t r0 = t.row == ALL_ROWS ? 0 : t.row, r1 = t.row == ALL_ROWS ? len : t.row + 1;
        for (size_t r = r0; r < r1; r++) for (int k = 0; k < d; k++) ev[r * d + k] = f_add(ev[r * d + k], t.delta[k]);
    }
}
// false when a tamper names nothing of this proof (a column, layer, row or byte that does not exist)
static bool tampers_fit(const Tampers& tp, size_t c, size_t aw, size_t kc, size_t N, size_t nf, size_t nl, size_t rs) {
    for (const Tamper& t : tp.list) {
        for (int k = 0; k < 3; k++) if (t.delta[k] >= P) return false;
        const bool all = t.row == ALL_ROWS;
        switch (t.target) {
            case T_MAIN_LDE: if (t.index >= c || (!all && t.row >= N)) return false; break;
            case T_AUX_LDE: if (t.index >= aw || (!all && t.row >= N)) return false; break;
            case T_CONSTRAINT_LDE: if (t.index >= kc || (!all && t.row >= N)) return false; break;
            case T_FRI_LAYER: {
                if (t.index > nl) return false;
                size_t len = N;
                for (u64 i = 0; i < t.index; i++) len /= nf;
                if (!all && t.row >= len) return false;
                break;
            }
            case T_REMAINDER: if (t.index >= rs || !all) return false; break;
            case T_REMAINDER_LONG: if (t.index < 1 || t.index > 64 || !all) return false; break;
            case T_FLIP_AUX: if (!aw) return false; break;
            case T_FLIP_FRI: if (t.index >= nl) return false; break;
            case T_FLIP_TRACE: case T_FLIP_CONSTRAINT: break;
            default: return false;
        }
    }
    return true;
}

struct StageTimer {
    bool on; double t0;
    StageTimer() : on(getenv("WFO_TIMING") != nullptr), t0(omp_get_wtime()) {}
    void mark(const char* name) { if (!on) return; double t = omp_get_wtime(); fprintf(stderr, "[oracle] %-26s %9.3f ms\n", name, (t - t0) * 1e3); t0 = t; }
};

static bool apply_aux_values(Air& air, const std::vector<EE>& rnd, int d) {
    if (!air.aux_values_fn) return true;
    size_t total = 0;
    for (auto& a : air.aux_asserts) total += a.values.size();
    std::vector<u64> rw(air.nr * d), vals(total * d);
    for (size_t i = 0; i < air.nr; i++) for (int k = 0; k < d; k++) rw[i * d + k] = rnd[i].v[k];
    size_t q = 0;
    for (auto& a : air.aux_asserts) for (auto& v : a.values) { for (int k = 0; k < d; k++) vals[q * d + k] = v.v[k]; q++; }
    if (air.aux_values_fn(air.aux_values_user, rw.data(), vals.data())) return false;
    q = 0;
    for (auto& a : air.aux_asserts)
        for (auto& v : a.values) {
            for (int k = 0; k < 3; k++) v.v[k] = k < d ? vals[q * d + k] : 0;
            for (int k = 0; k < d; k++) if (v.v[k] >= P) return false;
            q++;
        }
    return true;
}

// tp: the tampers of a dishonest proof (nullptr: an honest one); an empty result when one of them does not fit the proof
static std::vector<u8> prove_fib(const FibAir& air_in, const u64* trace /*[w][n]*/, AuxBuilder aux_builder = nullptr,
                                  void* aux_user = nullptr, Tampers* tp = nullptr) {
    FibAir air = air_in;  // the aux assertion values may be rewritten from the random elements (get_aux_assertions)
    StageTimer tm;
    const Opts& o = air.o;
    const int h = o.hash_id;
    Field F{(int)o.ext};
    const int d = F.d;
    const size_t n = air.n, N = air.lde_size(), c = air.width(), b = o.blowup, aw = air.aw;
    if (tp) {
        size_t nl = 0, dom = N, rs = n;
        while (dom > (size_t)(o.rem_max_deg + 1) * b) { dom /= o.folding; rs /= o.folding; nl++; }
        if (!tampers_fit(*tp, c, aw, air.num_comp_cols(), N, o.folding, nl, rs)) return {};
    }
    std::vector<u64> lde_t, alde_t, clde_t;   // the committed copies of tampered LDEs
    // channel (prover/src/channel.rs:57-82)
    std::vector<u64> seed = context_elements(air);
    for (u64 r : air.pub_inputs) seed.push_back(r);
    Coin coin(h, seed);
    Writer commitments;

    // 1. main trace commitment (lib.rs:497-522, trace_lde/default/mod.rs:245-282)
    std::vector<u64> polys(trace, trace + c * n);
    interpolate_columns(polys.data(), c, n, 1);
    std::vector<u64> lde(N * c);
    lde_rows(polys.data(), c, n, 1, b, lde.data());
    const u64* lde_c = committed(tp, T_MAIN_LDE, lde, N, c, 1, lde_t);
    std::vector<u8> t_leaves(N * 32), t_nodes(N * 32);
    hash_rows(h, lde_c, N, c, o.part_words(c, 1), t_leaves.data());  // row_matrix.rs:191 with E = BaseField
    merkle_nodes(h, t_leaves.data(), N, t_nodes.data());
    commitments.bytes(t_nodes.data() + 32, digest_len(h));
    coin.reseed(t_nodes.data() + 32);

    // 1b. auxiliary segment (lib.rs:309-349, air/src/air/mod.rs:292-306, trace_lde/default/mod.rs:140-166)
    std::vector<EE> rnd;
    std::vector<u64> apolys, alde;
    const u64* alde_c = nullptr;
    std::vector<u8> a_leaves, a_nodes;
    if (aw) {
        for (size_t i = 0; i < air.nr; i++) rnd.push_back(coin.draw(F));
        std::vector<u64> rw(air.nr * d);
        for (size_t i = 0; i < air.nr; i++) for (int k = 0; k < d; k++) rw[i * d + k] = rnd[i].v[k];
        apolys.assign(aw * n * d, 0);
        if (!aux_builder || aux_builder(aux_user, rw.data(), apolys.data())) abort();
        if (!apply_aux_values(air, rnd, d)) abort();
        interpolate_columns(apolys.data(), aw, n, d);
        alde.resize(N * aw * d);
        lde_rows(apolys.data(), aw, n, d, b, alde.data());
        alde_c = committed(tp, T_AUX_LDE, alde, N, aw, d, alde_t);
        a_leaves.resize(N * 32); a_nodes.resize(N * 32);
        hash_rows(h, alde_c, N, aw * d, o.part_words(aw, d), a_leaves.data());
        merkle_nodes(h, a_leaves.data(), N, a_nodes.data());
        commitments.bytes(a_nodes.data() + 32, digest_len(h));
        coin.reseed(a_nodes.data() + 32);
    }

    tm.mark("trace_commit");
    // 2. constraint evaluation (evaluator/default.rs:60-118, evaluation_table.rs:163-407)
    std::vector<EE> ccoef = coin.draw_coeffs(F, (int)o.batch_c, air.num_transition() + air.num_assertions());
    const CeEvaluator ev(air, d, ccoef, rnd.data());
    const size_t ce = n * air.ce_blowup();
    const size_t lde_shift = (size_t)__builtin_ctzll(b / air.ce_blowup());
    const u64 g_tr = root_of_unity((u32)__builtin_ctzll(n));
    std::vector<EE> comp(ce);
#pragma omp parallel
    {
        CeEvaluator::Scratch s = ev.scratch();
#pragma omp for schedule(static)
        for (size_t i = 0; i < ce; i++) {
            size_t ls = i << lde_shift, lx = (ls + b) % N;  // trace_lde/default/mod.rs:169-180
            comp[i] = ev.row(i, &lde[ls * c], &lde[lx * c], aw ? &alde[ls * aw * d] : nullptr, aw ? &alde[lx * aw * d] : nullptr, s);
        }
    }
    // 3. composition polynomial + commitment (composition_poly.rs:58-78, commitment/default.rs:109-150)
    std::vector<u64> cp(ce * d);
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < ce; i++) for (int k = 0; k < d; k++) cp[i * d + k] = comp[i].v[k];
    { auto itw = get_inv_twiddles(ce); interpolate_poly_with_offset(cp.data(), ce, d, itw.data(), GENERATOR); }
    const size_t kc = air.num_comp_cols();
    std::vector<u64> cpolys(kc * n * d);                      // column j = coefficients [j*n, (j+1)*n)
    for (size_t j = 0; j < kc; j++) memcpy(&cpolys[j * n * d], &cp[j * n * d], n * d * 8);
    std::vector<u64> clde(N * kc * d);
    lde_rows(cpolys.data(), kc, n, d, b, clde.data());
    const u64* clde_c = committed(tp, T_CONSTRAINT_LDE, clde, N, kc, d, clde_t);
    std::vector<u8> c_leaves(N * 32), c_nodes(N * 32);
    hash_rows(h, clde_c, N, kc * d, o.part_words(kc, d), c_leaves.data());
    merkle_nodes(h, c_leaves.data(), N, c_nodes.data());
    commitments.bytes(c_nodes.data() + 32, digest_len(h));
    coin.reseed(c_nodes.data() + 32);

    tm.mark("composition_commit");
    // 4. OOD frame (lib.rs:392-401, poly_table.rs:68-76, composition_poly.rs:101-108, channel.rs:102-113)
    EE z = coin.draw(F);
    EE zg = F.mul_base(z, g_tr);
    const size_t ct = c + aw;  // main columns then aux columns (ood_frame.rs:40-72)
    std::vector<EE> t_cur(ct), t_nxt(ct), q_cur(kc), q_nxt(kc);
    // ColMatrix::evaluate_columns_at (col_matrix.rs:245-252): iter!(columns) — parallel over columns in the `concurrent` build
#pragma omp parallel for schedule(dynamic, 1)
    for (size_t jj = 0; jj < 2 * c; jj++) {
        const size_t j = jj >> 1;
        if (jj & 1) t_nxt[j] = horner_base(F, &polys[j * n], n, zg); else t_cur[j] = horner_base(F, &polys[j * n], n, z);
    }
#pragma omp parallel for schedule(dynamic, 1)
    for (size_t j = 0; j < aw; j++) {
        std::vector<EE> pe(n);
        for (size_t i = 0; i < n; i++) { pe[i] = F.zero(); for (int k = 0; k < d; k++) pe[i].v[k] = apolys[(j * n + i) * d + k]; }
        t_cur[c + j] = horner_ext(F, pe.data(), n, z); t_nxt[c + j] = horner_ext(F, pe.data(), n, zg);
    }
#pragma omp parallel for schedule(dynamic, 1)
    for (size_t jj = 0; jj < 2 * kc; jj++) {
        const size_t j = jj >> 1;
        std::vector<EE> pe(n);
        for (size_t i = 0; i < n; i++) { pe[i] = F.zero(); for (int k = 0; k < d; k++) pe[i].v[k] = cpolys[(j * n + i) * d + k]; }
        if (jj & 1) q_nxt[j] = horner_ext(F, pe.data(), n, zg); else q_cur[j] = horner_ext(F, pe.data(), n, z);
    }
    Writer ood_t, ood_q;
    ood_t.u8_(2); ood_t.elems(F, t_cur.data(), ct); ood_t.elems(F, t_nxt.data(), ct); // ood_frame.rs:59-72
    ood_q.u8_(2); ood_q.elems(F, q_cur.data(), kc); ood_q.elems(F, q_nxt.data(), kc); // :95-108
    {
        std::vector<u64> m;  // merge_ood_evaluations ood_frame.rs:335-349
        auto push = [&](const std::vector<EE>& v) { for (auto& e : v) for (int k = 0; k < d; k++) m.push_back(e.v[k]); };
        push(t_cur); push(q_cur); push(t_nxt); push(q_nxt);
        u8 dg[32];
        hash_elements(h, m.data(), m.size(), dg);
        coin.reseed(dg);
    }
    tm.mark("ood_frames");
    // 5. DEEP composition polynomial, coefficient form (composer/mod.rs:67-210)
    std::vector<EE> dcoef = coin.draw_coeffs(F, (int)o.batch_d, ct + kc);
    std::vector<EE> comp_z(n, F.zero()), comp_gz(n, F.zero());
    for (size_t j = 0; j < c; j++) {  // acc_trace_poly: mul_acc (iter_mut!: parallel over i when `concurrent`) + constant term
#pragma omp parallel for schedule(static) if (n >= 1024)
        for (size_t i = 0; i < n; i++) {
            EE t = F.mul_base(dcoef[j], polys[j * n + i]);
            comp_z[i] = F.add(comp_z[i], t); comp_gz[i] = F.add(comp_gz[i], t);
        }
        comp_z[0] = F.sub(comp_z[0], F.mul(t_cur[j], dcoef[j]));
        comp_gz[0] = F.sub(comp_gz[0], F.mul(t_nxt[j], dcoef[j]));
    }
    for (size_t j = 0; j < aw; j++) {  // composer/mod.rs:100-125 aux trace polys, acc_trace_poly::<E, E>
#pragma omp parallel for schedule(static) if (n >= 1024)
        for (size_t i = 0; i < n; i++) {
            EE pe = F.zero(); for (int k = 0; k < d; k++) pe.v[k] = apolys[(j * n + i) * d + k];
            EE t = F.mul(pe, dcoef[c + j]);
            comp_z[i] = F.add(comp_z[i], t); comp_gz[i] = F.add(comp_gz[i], t);
        }
        comp_z[0] = F.sub(comp_z[0], F.mul(t_cur[c + j], dcoef[c + j]));
        comp_gz[0] = F.sub(comp_gz[0], F.mul(t_nxt[c + j], dcoef[c + j]));
    }
    for (size_t j = 0; j < kc; j++) {
#pragma omp parallel for schedule(static) if (n >= 1024)
        for (size_t i = 0; i < n; i++) {
            EE pe = F.zero(); for (int k = 0; k < d; k++) pe.v[k] = cpolys[(j * n + i) * d + k];
            EE t = F.mul(pe, dcoef[ct + j]);
            comp_z[i] = F.add(comp_z[i], t); comp_gz[i] = F.add(comp_gz[i], t);
        }
        comp_z[0] = F.sub(comp_z[0], F.mul(q_cur[j], dcoef[ct + j]));
        comp_gz[0] = F.sub(comp_gz[0], F.mul(q_nxt[j], dcoef[ct + j]));
    }
    auto syn_div = [&](std::vector<EE>& p, const EE& bb) {  // polynom/mod.rs:498-505 (a == 1)
        EE cc = F.zero();
        for (size_t i = p.size(); i-- > 0;) { p[i] = F.add(p[i], F.mul(bb, cc)); std::swap(p[i], cc); }
    };
    // merge_compositions (composer/mod.rs:186-200): iter_mut!(polys).zip(divisors) — the two divisions run side by side
#pragma omp parallel sections num_threads(2)
    {
#pragma omp section
        syn_div(comp_z, z);
#pragma omp section
        syn_div(comp_gz, zg);
    }
    std::vector<u64> deep(n * d);
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < n; i++) { EE s = F.add(comp_z[i], comp_gz[i]); for (int k = 0; k < d; k++) deep[i * d + k] = s.v[k]; }
    std::vector<u64> deep_ev(N * d);
    { auto tw = get_twiddles(n); evaluate_poly_with_offset(deep.data(), n, d, tw.data(), GENERATOR, b, deep_ev.data()); }

    tm.mark("deep_composition");
    // 6. FRI commit phase with the prover channel (fri/src/prover/mod.rs:179-239, channel.rs:215-234)
    struct Layer { std::vector<u64> tv; std::vector<u8> leaves, nodes; size_t rows; };
    std::vector<Layer> layers;
    std::vector<u64> cur(deep_ev);
    size_t cur_len = N;
    const size_t nf = o.folding, max_rem = (size_t)(o.rem_max_deg + 1) * b;
    while (cur_len > max_rem) {
        tamper_layer(tp, layers.size(), cur, cur_len, d);
        Layer L;
        L.rows = cur_len / nf;
        L.tv.resize(cur_len * d);
        transpose_slice(cur.data(), cur_len, d, nf, L.tv.data());
        L.leaves.resize(L.rows * 32); L.nodes.resize(L.rows * 32);
        hash_rows(h, L.tv.data(), L.rows, nf * d, nf * d, L.leaves.data());
        merkle_nodes(h, L.leaves.data(), L.rows, L.nodes.data());
        commitments.bytes(L.nodes.data() + 32, digest_len(h));
        coin.reseed(L.nodes.data() + 32);
        EE alpha = coin.draw(F);
        std::vector<u64> nxt(L.rows * d);
        apply_drp(L.tv.data(), L.rows, d, nf, GENERATOR, alpha.v, nxt.data());
        cur.swap(nxt);
        cur_len = L.rows;
        layers.push_back(std::move(L));
    }
    std::vector<u64> remainder;
    {
        tamper_layer(tp, layers.size(), cur, cur_len, d);
        auto itw = get_inv_twiddles(cur_len);
        interpolate_poly_with_offset(cur.data(), cur_len, d, itw.data(), GENERATOR);
        size_t rs = cur_len / b;
        remainder.resize(rs * d);
        for (size_t i = 0; i < rs; i++) for (int k = 0; k < d; k++) remainder[i * d + k] = cur[(rs - 1 - i) * d + k];
        if (tp)
            for (const Tamper& t : tp->list) {
                if (t.target == T_REMAINDER)
                    for (int k = 0; k < d; k++) remainder[t.index * d + k] = f_add(remainder[t.index * d + k], t.delta[k]);
                if (t.target == T_REMAINDER_LONG) remainder.insert(remainder.begin(), t.index * d, 0);
            }
        u8 dg[32];
        hash_elements(h, remainder.data(), remainder.size(), dg);
        commitments.bytes(dg, digest_len(h));
        coin.reseed(dg);
    }
    tm.mark("fri_layers");
    // 7. grinding + query positions (channel.rs:151-184; serial branch: smallest nonce)
    u64 nonce = 1;
    while (wfo_coin_leading_zeros(&coin.c, nonce) < o.grinding) nonce++;
    std::vector<u64> pos(o.num_queries);
    if (wfo_coin_draw_integers(&coin.c, o.num_queries, N, nonce, pos.data())) abort();
    std::sort(pos.begin(), pos.end());
    pos.erase(std::unique(pos.begin(), pos.end()), pos.end());

    tm.mark("grinding");
    // 8. proof object (lib.rs:464-489; air/src/proof/mod.rs:189-200)
    Writer w;
    write_context(w, air);
    w.u8_((u8)pos.size());
    w.u16_((uint16_t)commitments.b.size()); w.bytes(commitments.b.data(), commitments.b.size());
    std::vector<Section> sec(T_FLIP_FRI + layers.size());   // opened values of T_FLIP_TRACE .. T_FLIP_FRI + layer
    sec[T_FLIP_TRACE] = queries_for(F, h, lde_c, c, t_leaves, t_nodes, N, pos, w);          // trace queries: main segment
    if (aw) sec[T_FLIP_AUX] = queries_for(F, h, alde_c, aw * d, a_leaves, a_nodes, N, pos, w);  // aux segment (trace_lde/default/mod.rs:199-218)
    sec[T_FLIP_CONSTRAINT] = queries_for(F, h, clde_c, kc * d, c_leaves, c_nodes, N, pos, w);    // constraint queries
    w.u16_((uint16_t)ood_t.b.size()); w.bytes(ood_t.b.data(), ood_t.b.size());
    w.u16_((uint16_t)ood_q.b.size()); w.bytes(ood_q.b.data(), ood_q.b.size());
    // FriProof (fri/src/prover/mod.rs:254-319, fri/src/proof.rs:149-163,275-285)
    w.u8_((u8)layers.size());
    {
        std::vector<u64> p = pos;
        size_t dom = N;
        for (auto& L : layers) {
            std::vector<u64> fp(p.size());
            size_t nfp = fold_positions(p.data(), p.size(), dom, nf, fp.data());
            fp.resize(nfp);
            p = fp;
            Writer vals;
            for (u64 q : p) vals.bytes(&L.tv[q * nf * d], nf * d * 8);
            std::vector<u8> lv(p.size() * 32), pr(64 + p.size() * 40 * 33);
            long pl = merkle_prove_batch(L.leaves.data(), L.nodes.data(), L.rows, p.data(), p.size(), lv.data(), pr.data(), pr.size(), digest_len(h));
            if (pl < 0) abort();
            w.u32_((u32)vals.b.size());
            sec[T_FLIP_FRI + (&L - layers.data())] = Section{w.b.size(), vals.b.size()};
            w.bytes(vals.b.data(), vals.b.size());
            w.u32_((u32)pl); w.bytes(pr.data(), (size_t)pl);
            dom /= nf;
        }
    }
    w.u16_((uint16_t)(remainder.size() * 8)); w.bytes(remainder.data(), remainder.size() * 8);
    w.u8_(0);
    w.u64_(nonce);
    tm.mark("queries_and_proof");
    if (tp) {
        for (const Tamper& t : tp->list) {
            if (t.target < T_FLIP_TRACE) continue;
            const Section s = sec[t.target == T_FLIP_FRI ? T_FLIP_FRI + t.index : t.target];
            const u64 at = t.row == ALL_ROWS ? 0 : t.row;
            if (at >= s.len) return {};
            w.b[s.off + at] ^= (u8)(1u << (t.delta[0] & 7));
        }
        tp->positions = pos;
    }
    return w.b;
}

// =================================================================================================
// VERIFIER (verifier/src/lib.rs:82-260)
// =================================================================================================
struct Reader {
    const u8* p; size_t n, pos = 0; bool ok = true;
    u8 u8_() { if (pos + 1 > n) { ok = false; return 0; } return p[pos++]; }
    u64 le(int k) { u64 v = 0; if (pos + k > n) { ok = false; return 0; } for (int i = 0; i < k; i++) v |= (u64)p[pos + i] << (8 * i); pos += k; return v; }
    const u8* take(size_t k) { if (pos + k > n) { ok = false; return nullptr; } const u8* q = p + pos; pos += k; return q; }
    u64 usize() {  // vint64 (utils/core/src/serde/byte_reader.rs read_usize)
        if (pos >= n) { ok = false; return 0; }
        u8 first = p[pos];
        int len = first == 0 ? 9 : __builtin_ctz(first) + 1;
        if (pos + len > n) { ok = false; return 0; }
        u64 v;
        if (len == 9) { pos += 1; v = le(8); }
        else { u64 raw = 0; for (int i = 0; i < len; i++) raw |= (u64)p[pos + i] << (8 * i); pos += len; v = raw >> len; }
        return v;
    }
};

// ElementDigest::read_from (rp64_256/digest.rs:61-69, rp64_256_jive/digest.rs:61-69) reads each digest word through
// BaseElement::new, which reduces a word w >= p to w - p: a Rescue commitment or Merkle path node stands for its reduced digest.
// ByteDigest (BLAKE3, SHA3) is taken as it is.
static void reduce_digest(int h, u8* dg) {
    if (h != WFO_HASH_RP64_256 && h != WFO_HASH_RPJIVE64_256) return;
    for (int k = 0; k < 4; k++) { u64 w; memcpy(&w, dg + 8 * k, 8); if (w >= P) w -= P; memcpy(dg + 8 * k, &w, 8); }
}
// BaseElement::read_from refuses a word >= p (math/src/field/f64/mod.rs:673-681)
static bool words_canonical(const u8* b, size_t len) {
    for (size_t at = 0; at + 8 <= len; at += 8) { u64 w; memcpy(&w, b + at, 8); if (w >= P) return false; }
    return true;
}

struct BatchProof { u8 depth; std::vector<std::vector<std::array<u8, 32>>> nodes; };
static bool read_batch_proof(Reader& r, BatchProof& bp, int h) {
    const size_t dlen = digest_len(h);
    bp.depth = r.u8_();
    u64 nv = r.usize();
    if (!r.ok || nv > 100000 || bp.depth < 1 || bp.depth > 40) return false;   // a tree of 2^depth leaves; callers shift by it
    bp.nodes.resize(nv);
    for (auto& v : bp.nodes) {
        u64 ln = r.usize();
        if (!r.ok || ln > 64) return false;
        v.resize(ln);
        for (auto& dg : v) { const u8* q = r.take(dlen); if (!q) return false; dg.fill(0); memcpy(dg.data(), q, dlen); reduce_digest(h, dg.data()); }
    }
    return r.ok;
}
// BatchMerkleProof::get_root (crypto/src/merkle/proofs.rs:90-205)
static bool batch_root(int h, const BatchProof& bp, const std::vector<u64>& indexes, const std::vector<std::array<u8, 32>>& leaves,
                       u8 root[32]) {
    if (indexes.empty() || indexes.size() != leaves.size()) return false;
    std::map<size_t, size_t> index_map;
    size_t nl = (size_t)1 << bp.depth;
    for (size_t i = 0; i < indexes.size(); i++) { if (indexes[i] >= nl) return false; index_map[indexes[i]] = i; }
    if (index_map.size() != indexes.size()) return false;
    std::set<size_t> norm;
    for (u64 i : indexes) norm.insert(i & ~(size_t)1);
    if (norm.size() != bp.nodes.size()) return false;
    std::map<size_t, std::array<u8, 32>> v;
    std::vector<size_t> next, ptr;
    size_t i = 0;
    for (size_t index : norm) {
        u8 buf[64];
        auto a = index_map.find(index), b2 = index_map.find(index + 1);
        if (a != index_map.end()) {
            memcpy(buf, leaves[a->second].data(), 32);
            if (b2 != index_map.end()) { memcpy(buf + 32, leaves[b2->second].data(), 32); ptr.push_back(0); }
            else { if (bp.nodes[i].empty()) return false; memcpy(buf + 32, bp.nodes[i][0].data(), 32); ptr.push_back(1); }
        } else {
            if (bp.nodes[i].empty() || b2 == index_map.end()) return false;
            memcpy(buf, bp.nodes[i][0].data(), 32);
            memcpy(buf + 32, leaves[b2->second].data(), 32);
            ptr.push_back(1);
        }
        std::array<u8, 32> parent;
        merge(h, buf, parent.data());
        size_t pi = (nl + index) >> 1;
        v[pi] = parent;
        next.push_back(pi);
        i++;
    }
    for (int lvl = 1; lvl < bp.depth; lvl++) {
        std::vector<size_t> idx = next;
        next.clear();
        size_t q = 0;
        while (q < idx.size()) {
            size_t node_index = idx[q], sib_index = node_index ^ 1;
            std::array<u8, 32> sib;
            size_t slot = q;
            if (q + 1 < idx.size() && idx[q + 1] == sib_index) {
                auto it = v.find(sib_index);
                if (it == v.end()) return false;
                sib = it->second;
                q += 1;
            } else {
                if (bp.nodes[slot].size() <= ptr[slot]) return false;
                sib = bp.nodes[slot][ptr[slot]];
                ptr[slot] += 1;
            }
            auto nit = v.find(node_index);
            if (nit == v.end()) return false;
            u8 buf[64];
            if (node_index & 1) { memcpy(buf, sib.data(), 32); memcpy(buf + 32, nit->second.data(), 32); }
            else { memcpy(buf, nit->second.data(), 32); memcpy(buf + 32, sib.data(), 32); }
            std::array<u8, 32> parent;
            merge(h, buf, parent.data());
            v[node_index >> 1] = parent;
            next.push_back(node_index >> 1);
            q += 1;
        }
    }
    auto it = v.find(1);
    if (it == v.end()) return false;
    memcpy(root, it->second.data(), 32);
    return true;
}

enum { V_OK = 0, V_MALFORMED = 1, V_OOD = 2, V_POW = 3, V_TRACE_QUERY = 4, V_CONSTRAINT_QUERY = 5, V_FRI_LAYER = 6,
       V_FRI_FOLD = 7, V_FRI_REMAINDER = 8, V_CONTEXT = 9 };

static int verify_fib(const u8* proof, size_t len, FibAir air /* options + results filled by caller */) {
    Reader r{proof, len};
    // Context
    u8 mw = r.u8_(), aw = r.u8_(), ar = r.u8_(), logn = r.u8_();
    u64 meta = r.le(2);
    r.take(meta);
    u8 ml = r.u8_();
    const u8* mod = r.take(ml);
    if (!r.ok || ml != 8 || memcmp(mod, &P, 8) || aw != air.aw || ar != air.nr) return V_CONTEXT;
    Opts o = air.o;
    o.num_queries = r.u8_(); o.blowup = r.u8_(); o.grinding = r.u8_(); o.ext = r.u8_(); o.folding = r.u8_();
    o.rem_max_deg = r.u8_(); o.batch_c = r.u8_(); o.batch_d = r.u8_(); o.num_partitions = r.u8_(); o.hash_rate = r.u8_();
    u64 ncons = r.usize();
    if (!r.ok) return V_MALFORMED;
    // what deserialisation refuses in the reference: ProofOptions::new / with_partitions assert these ranges
    // (air/src/options.rs:143-172, :410-417), FieldExtension / BatchingMethod::read_from accept 1..=3 / 0..=2,
    // TraceInfo::read_from needs 2^logn >= 8 (trace_info.rs MIN_TRACE_LENGTH) and the LDE domain must fit the field's
    // two-adicity (2^32 for f64, get_root_of_unity)
    auto pow2 = [](u64 v) { return v && !(v & (v - 1)); };
    if (o.num_queries == 0 || !pow2(o.blowup) || o.blowup < 2 || o.blowup > 128 || o.grinding > 32 || !pow2(o.folding) || o.folding < 2 ||
        o.folding > 16 || !pow2((u64)o.rem_max_deg + 1) || o.batch_c > 2 || o.batch_d > 2 || o.num_partitions < 1 || o.num_partitions > 16 ||
        o.hash_rate < 1)
        return V_MALFORMED;
    {
        u32 lb = 0;
        while ((1u << lb) < o.blowup) lb++;
        if (logn < 3 || logn + lb > 32) return V_MALFORMED;
    }
    air.o = o;
    air.n = (size_t)1 << logn;
    if (air.asserts.empty() && air.w > 0) {  // FibSmall x k entry point: assertions reference step n - 1
        std::vector<u64> res = air.pub_inputs;
        air = fib_air(air.w / 2, air.n, res.data(), o);
    }
    if (mw != air.width() || ncons != air.num_assertions() + air.num_transition() || o.ext < 1 || o.ext > 3) return V_CONTEXT;
    const int h = o.hash_id;
    Field F{(int)o.ext};
    const int d = F.d;
    const size_t n = air.n, N = air.lde_size(), c = air.width(), kc = air.num_comp_cols(), nf = o.folding, ct = c + air.aw;
    const size_t nseg = air.aw ? 2 : 1;
    u8 nuq = r.u8_();
    u64 clen = r.le(2);
    const u8* cm = r.take(clen);
    if (!r.ok) return V_MALFORMED;
    size_t nlayers = 0;
    { size_t dom = N, max_rem = (size_t)(o.rem_max_deg + 1) * o.blowup; while (dom > max_rem) { dom /= nf; nlayers++; } }
    const size_t dl = digest_len(h), ncm = nseg + 1 + nlayers + 1;
    if (clen != dl * ncm) return V_MALFORMED;
    std::vector<u8> cm32(32 * ncm, 0);   // the commitments in 32-byte slots (zero padded, as ByteDigest::as_bytes)
    for (size_t i = 0; i < ncm; i++) { memcpy(cm32.data() + 32 * i, cm + dl * i, dl); reduce_digest(h, cm32.data() + 32 * i); }
    cm = cm32.data();
    const u8* trace_root = cm; const u8* aux_root = cm + 32;  // air/src/proof/commitments.rs:66-100
    const u8* cons_root = cm + 32 * nseg; const u8* fri_roots = cm + 32 * (nseg + 1);
    // queries
    auto read_q = [&](std::vector<u8>& vals, std::vector<u8>& pr) {
        u64 vl = r.usize(); const u8* v = r.take(vl); if (!r.ok) return false; vals.assign(v, v + vl);
        u64 pl = r.usize(); const u8* p2 = r.take(pl); if (!r.ok) return false; pr.assign(p2, p2 + pl);
        return true;
    };
    std::vector<u8> tq_vals, tq_pr, aq_vals, aq_pr, cq_vals, cq_pr;
    if (!read_q(tq_vals, tq_pr) || (air.aw && !read_q(aq_vals, aq_pr)) || !read_q(cq_vals, cq_pr)) return V_MALFORMED;
    u64 otl = r.le(2); const u8* ot = r.take(otl);
    u64 oql = r.le(2); const u8* oq = r.take(oql);
    if (!r.ok || otl != 1 + 2 * ct * d * 8 || oql != 1 + 2 * kc * d * 8 || ot[0] != 2 || oq[0] != 2) return V_MALFORMED;
    auto rd = [&](const u8* p, size_t idx) { EE e = F.zero(); memcpy(e.v, p + idx * d * 8, d * 8); return e; };
    std::vector<EE> t_cur(ct), t_nxt(ct), q_cur(kc), q_nxt(kc);
    for (size_t j = 0; j < ct; j++) { t_cur[j] = rd(ot + 1, j); t_nxt[j] = rd(ot + 1, ct + j); }
    for (size_t j = 0; j < kc; j++) { q_cur[j] = rd(oq + 1, j); q_nxt[j] = rd(oq + 1, kc + j); }
    // FRI proof
    u8 fl = r.u8_();
    if (fl != nlayers) return V_MALFORMED;
    std::vector<std::vector<u8>> fv(fl), fp(fl);
    for (int i = 0; i < fl; i++) {
        u64 vl = r.le(4); const u8* v = r.take(vl); if (!r.ok) return V_MALFORMED; fv[i].assign(v, v + vl);
        u64 pl = r.le(4); const u8* p2 = r.take(pl); if (!r.ok) return V_MALFORMED; fp[i].assign(p2, p2 + pl);
    }
    u64 reml = r.le(2); const u8* rem = r.take(reml);
    const u8 fri_log_parts = r.u8_();   // FriProof::num_partitions, stored as a power of two (fri/src/proof.rs:36,101-103)
    u64 nonce = r.le(8);
    if (!r.ok || r.pos != len || reml % (8 * d)) return V_MALFORMED;
    // VerifierChannel::new (verifier/src/channel.rs:92-118) reads every field element of the proof with BaseElement::read_from
    // and turns a word >= p into ProofDeserializationError: the opened values (air/src/proof/table.rs:60-65), the OOD frames
    // (ood_frame.rs:140,157, after their frame-size byte), the FRI layer values and the remainder (fri/src/proof.rs:185,321)
    {
        bool ok = words_canonical(tq_vals.data(), tq_vals.size()) && words_canonical(aq_vals.data(), aq_vals.size()) &&
                  words_canonical(cq_vals.data(), cq_vals.size()) && words_canonical(ot + 1, otl - 1) && words_canonical(oq + 1, oql - 1) &&
                  words_canonical(rem, reml);
        for (auto& v : fv) ok = ok && words_canonical(v.data(), v.size());
        if (!ok) return V_MALFORMED;
    }

    // transcript (lib.rs:149-260)
    std::vector<u64> seed = context_elements(air);
    for (u64 x : air.pub_inputs) seed.push_back(x);
    Coin coin(h, seed);
    coin.reseed(trace_root);
    std::vector<EE> rnd;
    if (air.aw) {  // verifier/src/lib.rs:170-184
        for (size_t i = 0; i < air.nr; i++) rnd.push_back(coin.draw(F));
        coin.reseed(aux_root);
        if (!apply_aux_values(air, rnd, F.d)) return V_MALFORMED;   // Air::get_aux_assertions(aux_rand_elements)
    }
    std::vector<EE> ccoef = coin.draw_coeffs(F, (int)o.batch_c, air.num_transition() + air.num_assertions());
    coin.reseed(cons_root);
    EE z = coin.draw(F);
    // OOD consistency (verifier/src/evaluator.rs:15-80)
    {
        const size_t nTm = air.num_main_transition(), nT = air.num_transition();
        std::vector<EE> tcoef(ccoef.begin(), ccoef.begin() + nT);
        std::vector<EE> bcoef(ccoef.begin() + nT, ccoef.begin() + nT + air.asserts.size());
        std::vector<EE> tev(nT, F.zero());
        // periodic values at z: poly_j(z^(n/L_j)) (verifier/src/evaluator.rs:27-35)
        std::vector<EE> per;
        for (auto& poly : air.periodic_polys()) per.push_back(horner_base(F, poly.data(), poly.size(), F.exp(z, n / poly.size())));
        air.eval_transition(t_cur.data(), t_nxt.data(), per.data(), tev.data(),
                            [&](const EE& a, const EE& b) { return F.sub(a, b); }, [&](const EE& a, const EE& b) { return F.add(a, b); },
                            [&](const EE& a, const EE& b) { return F.mul(a, b); }, [&](u64 v) { return F.from_base(v); });
        if (air.aw)  // verifier/src/evaluator.rs:43-57
            air.eval_aux_transition(t_cur.data(), t_nxt.data(), t_cur.data() + c, t_nxt.data() + c, per.data(), rnd.data(),
                                    tev.data() + nTm, [&](const EE& a, const EE& b) { return F.sub(a, b); },
                                    [&](const EE& a, const EE& b) { return F.add(a, b); },
                                    [&](const EE& a, const EE& b) { return F.mul(a, b); }, [&](u64 v) { return F.from_base(v); });
        EE t = F.zero();
        for (size_t j = 0; j < tev.size(); j++) t = F.add(t, F.mul(tcoef[j], tev[j]));
        // transition divisor (x^n - 1) / prod (x - exemption) at z (transition/mod.rs:153-174, divisor.rs:79-100)
        EE num = F.sub(F.exp(z, n), F.one());
        EE den = F.one();
        for (u64 e : exemption_points(air)) den = F.mul(den, F.sub(z, F.from_base(e)));
        EE res = F.mul(t, F.mul(den, F.inv(num)));
        for (auto& G : boundary_groups(air, bcoef)) {
            EE bs = F.zero();
            for (auto& e : G.e)  // BoundaryConstraint::evaluate_at (air/src/air/boundary/constraint.rs:128-147)
                bs = F.add(bs, F.mul(F.sub(t_cur[e.col], horner_ext(F, e.poly.data(), e.poly.size(), F.mul_base(z, e.x_offset))), e.cc));
            res = F.add(res, F.mul(bs, F.inv(F.sub(F.exp(z, G.a), F.from_base(G.b)))));
        }
        for (auto& G : aux_boundary_groups(air, ccoef.data() + nT + air.asserts.size())) {  // evaluator.rs:76-83
            EE bs = F.zero();
            for (auto& e : G.e)
                bs = F.add(bs, F.mul(F.sub(t_cur[c + e.col], horner_ext(F, e.poly.data(), e.poly.size(), F.mul_base(z, e.x_offset))), e.cc));
            res = F.add(res, F.mul(bs, F.inv(F.sub(F.exp(z, G.a), F.from_base(G.b)))));
        }
        EE res2 = F.zero();
        for (size_t i = 0; i < kc; i++) res2 = F.add(res2, F.mul(F.exp(z, i * n), q_cur[i]));
        if (!F.eq(res, res2)) return V_OOD;
    }
    {
        std::vector<u64> m;
        auto push = [&](const std::vector<EE>& v) { for (auto& e : v) for (int k = 0; k < d; k++) m.push_back(e.v[k]); };
        push(t_cur); push(q_cur); push(t_nxt); push(q_nxt);
        u8 dg[32];
        hash_elements(h, m.data(), m.size(), dg);
        coin.reseed(dg);
    }
    std::vector<EE> dcoef = coin.draw_coeffs(F, (int)o.batch_d, ct + kc);
    // FriVerifier::new (fri/src/verifier/mod.rs:48-90): reseed + draw for every commitment incl. remainder
    std::vector<EE> alphas;
    for (size_t i = 0; i <= nlayers; i++) { coin.reseed(fri_roots + 32 * i); alphas.push_back(coin.draw(F)); }
    if (wfo_coin_leading_zeros(&coin.c, nonce) < o.grinding) return V_POW;
    std::vector<u64> pos(o.num_queries);
    if (wfo_coin_draw_integers(&coin.c, o.num_queries, N, nonce, pos.data())) return V_MALFORMED;
    std::sort(pos.begin(), pos.end());
    pos.erase(std::unique(pos.begin(), pos.end()), pos.end());
    if (pos.size() != nuq) return V_MALFORMED;
    // trace / constraint queries (verifier/src/channel.rs:206-260)
    // hash_row (verifier/src/channel.rs:431-453): rows are re-hashed in partitions of `part` base elements
    auto check_q = [&](const std::vector<u8>& vals, const std::vector<u8>& pr, size_t row_words, size_t part, const u8* root) {
        if (vals.size() != pos.size() * row_words * 8) return false;
        std::vector<std::array<u8, 32>> lv(pos.size());
        for (size_t i = 0; i < pos.size(); i++) hash_rows(h, (const u64*)(vals.data() + i * row_words * 8), 1, row_words, part, lv[i].data());
        Reader pr_r{pr.data(), pr.size()};
        BatchProof bp;
        if (!read_batch_proof(pr_r, bp, h) || pr_r.pos != pr.size() || ((size_t)1 << bp.depth) != N) return false;
        u8 got[32];
        return batch_root(h, bp, pos, lv, got) && !memcmp(got, root, 32);
    };
    if (!check_q(tq_vals, tq_pr, c, o.part_words(c, 1), trace_root)) return V_TRACE_QUERY;
    if (air.aw && !check_q(aq_vals, aq_pr, air.aw * d, o.part_words(air.aw, d), aux_root)) return V_TRACE_QUERY;  // channel.rs:206-240
    if (!check_q(cq_vals, cq_pr, kc * d, o.part_words(kc, d), cons_root)) return V_CONSTRAINT_QUERY;
    // DEEP composition at the query positions (verifier/src/composer.rs)
    u64 g_lde = root_of_unity((u32)__builtin_ctzll(N)), g_tr = root_of_unity((u32)__builtin_ctzll(n));
    EE zg = F.mul_base(z, g_tr);
    std::vector<EE> evals(pos.size());
    for (size_t qi = 0; qi < pos.size(); qi++) {
        EE x = F.from_base(f_mul(f_exp(g_lde, pos[qi]), GENERATOR));
        const u64* trow = (const u64*)(tq_vals.data() + qi * c * 8);
        const u64* crow = (const u64*)(cq_vals.data() + qi * kc * d * 8);
        EE t1 = F.zero(), t2 = F.zero();
        for (size_t j = 0; j < c; j++) {
            EE v = F.from_base(trow[j]);
            t1 = F.add(t1, F.mul(F.sub(v, t_cur[j]), dcoef[j]));
            t2 = F.add(t2, F.mul(F.sub(v, t_nxt[j]), dcoef[j]));
        }
        for (size_t j = 0; j < air.aw; j++) {  // composer.rs:103-130
            EE v = F.zero(); memcpy(v.v, aq_vals.data() + (qi * air.aw + j) * d * 8, d * 8);
            t1 = F.add(t1, F.mul(F.sub(v, t_cur[c + j]), dcoef[c + j]));
            t2 = F.add(t2, F.mul(F.sub(v, t_nxt[c + j]), dcoef[c + j]));
        }
        for (size_t j = 0; j < kc; j++) {
            EE v = F.zero(); memcpy(v.v, crow + j * d, d * 8);
            t1 = F.add(t1, F.mul(F.sub(v, q_cur[j]), dcoef[ct + j]));
            t2 = F.add(t2, F.mul(F.sub(v, q_nxt[j]), dcoef[ct + j]));
        }
        EE d1 = F.sub(x, z), d2 = F.sub(x, zg);
        evals[qi] = F.mul(F.add(F.mul(t1, d2), F.mul(t2, d1)), F.inv(F.mul(d1, d2)));
    }
    // FRI verification (fri/src/verifier/mod.rs:210-331)
    {
        std::vector<u64> positions = pos;
        size_t dom = N;
        u64 dg = g_lde;
        for (size_t depth = 0; depth < nlayers; depth++) {
            std::vector<u64> fpos(positions.size());
            fpos.resize(fold_positions(positions.data(), positions.size(), dom, nf, fpos.data()));
            // map_positions_to_indexes (fri/src/utils.rs:9-33): with P = 2^fri_log_parts > 1 partitions the verifier looks the
            // folded positions up at index (p mod P) (target / P) + (p - p mod P) / P of the layer commitment. The prover this
            // oracle restates commits every layer in domain order (P = 1): any other index set cannot open that commitment.
            if (fri_log_parts) {
                if (fri_log_parts >= 32) return V_MALFORMED;
                const u64 P_ = (u64)1 << fri_log_parts, target = dom / nf, psize = target / P_;
                for (u64 p : fpos)
                    if ((p % P_) * psize + (p - p % P_) / P_ != p) return V_FRI_LAYER;
            }
            const std::vector<u8>& vals = fv[depth];
            if (vals.size() != fpos.size() * nf * d * 8) return V_FRI_LAYER;
            std::vector<std::array<u8, 32>> lv(fpos.size());
            for (size_t i = 0; i < fpos.size(); i++) hash_elements(h, (const u64*)(vals.data() + i * nf * d * 8), nf * d, lv[i].data());
            Reader pr_r{fp[depth].data(), fp[depth].size()};
            BatchProof bp;
            if (!read_batch_proof(pr_r, bp, h) || pr_r.pos != fp[depth].size() || ((size_t)1 << bp.depth) != dom / nf) return V_FRI_LAYER;
            u8 got[32];
            if (!batch_root(h, bp, fpos, lv, got) || memcmp(got, fri_roots + 32 * depth, 32)) return V_FRI_LAYER;
            // get_query_values
            size_t row_len = dom / nf;
            for (size_t i = 0; i < positions.size(); i++) {
                size_t idx = std::find(fpos.begin(), fpos.end(), positions[i] % row_len) - fpos.begin();
                EE v = F.zero();
                memcpy(v.v, vals.data() + (idx * nf + positions[i] / row_len) * d * 8, d * 8);
                if (!F.eq(v, evals[i])) return V_FRI_FOLD;
            }
            // fold each queried row: interpolate over {x_e * w_nf^r} and evaluate at alpha — the same
            // value apply_drp computes (folding/mod.rs:86-118)
            std::vector<EE> nxt(fpos.size());
            for (size_t i = 0; i < fpos.size(); i++) {
                std::vector<u64> row(nf * d), o2(d);
                memcpy(row.data(), vals.data() + i * nf * d * 8, nf * d * 8);
                // apply_drp on a single row needs x = offset * g^pos: emulate with the row's inverse offset
                u64 xinv = f_inv(f_mul(f_exp(dg, fpos[i]), GENERATOR));
                auto itw = get_inv_twiddles(nf);
                ref_fft_in_place(row.data(), nf, d, itw.data());
                permute_words(row.data(), nf, d);
                u64 off = f_inv((u64)nf);
                EE acc = F.zero();
                std::vector<EE> coefs(nf);
                for (size_t j = 0; j < nf; j++) {
                    coefs[j] = F.zero();
                    for (int k = 0; k < d; k++) coefs[j].v[k] = f_mul(row[j * d + k], off);
                    off = f_mul(off, xinv);
                }
                acc = horner_ext(F, coefs.data(), nf, alphas[depth]);
                nxt[i] = acc;
            }
            evals = nxt;
            positions = fpos;
            dg = f_exp(dg, nf);
            dom /= nf;
        }
        size_t rn = reml / (8 * d), mdp1 = n;   // max_degree_plus_1 after folding (verifier/mod.rs:296-300)
        for (size_t i = 0; i < nlayers; i++) mdp1 /= nf;
        if (rn > mdp1) return V_FRI_REMAINDER;
        for (size_t i = 0; i < positions.size(); i++) {
            u64 x = f_mul(f_exp(dg, positions[i]), GENERATOR);
            EE acc = F.zero();
            for (size_t j = 0; j < rn; j++) {  // eval_horner_rev
                EE cj = F.zero(); memcpy(cj.v, rem + j * d * 8, d * 8);
                acc = F.add(F.mul_base(acc, x), cj);
            }
            if (!F.eq(acc, evals[i])) return V_FRI_REMAINDER;
        }
    }
    return V_OK;
}

}  // namespace

extern "C" {
// opts: [num_queries, blowup, grinding, ext, folding, rem_max_deg, batch_constraints, batch_deep,
//        hash_id | num_partitions << 8 | hash_rate << 16]  (ProofOptions::with_partitions, air/src/options.rs:193-200;
//        0 in either partition field = the default PartitionOptions::new(1, 1))
static Opts make_opts(const uint32_t* v) {
    Opts o;
    o.num_queries = v[0]; o.blowup = v[1]; o.grinding = v[2]; o.ext = v[3]; o.folding = v[4]; o.rem_max_deg = v[5];
    o.batch_c = v[6]; o.batch_d = v[7]; o.hash_id = (int)(v[8] & 0xff);
    o.num_partitions = (v[8] >> 8) & 0xff; o.hash_rate = (v[8] >> 16) & 0xff;
    if (o.num_partitions == 0) o.num_partitions = 1;
    if (o.hash_rate == 0) o.hash_rate = 1;
    return o;
}
// Every proving entry point ends in these arguments: `tamper` [ntamper][6] words {target, index, row, delta[3]} (the
// Tamper list of a dishonest proof, see T_* above; ntamper = 0 for an honest proof) and, when `positions` is not null,
// the query positions the proof opens (at most num_queries words) with their count in *npositions.
static long prove_entry(const Air& air, const uint64_t* trace, AuxBuilder builder, void* user, const uint64_t* tamper,
                        size_t ntamper, uint64_t* positions, size_t* npositions, uint8_t* out, size_t cap) {
    Tampers tp;
    for (size_t i = 0; i < ntamper; i++) {
        const uint64_t* t = tamper + 6 * i;
        tp.list.push_back(Tamper{t[0], t[1], t[2], {t[3], t[4], t[5]}});
    }
    std::vector<u8> p = prove_fib(air, trace, builder, user, ntamper || positions ? &tp : nullptr);
    if (p.empty()) return -4;
    if (p.size() > cap) return -1;
    memcpy(out, p.data(), p.size());
    if (positions) {
        memcpy(positions, tp.positions.data(), tp.positions.size() * 8);
        *npositions = tp.positions.size();
    }
    return (long)p.size();
}
// trace: [2k][n] canonical words; results: k words. Returns proof length (bytes written to out), -1 when it does not fit,
// -4 for a tamper that does not fit the proof.
long wfo_prove_fib(const uint64_t* trace, size_t k, size_t n, const uint64_t* results, const uint32_t* opts, uint8_t* out,
                   size_t cap, const uint64_t* tamper, size_t ntamper, uint64_t* positions, size_t* npositions) {
    Air air = fib_air(k, n, results, make_opts(opts));
    return prove_entry(air, trace, nullptr, nullptr, tamper, ntamper, positions, npositions, out, cap);
}
// 0 = accepted; otherwise the failed check (V_* above)
int wfo_verify_fib(const uint8_t* proof, size_t len, size_t k, const uint64_t* results, int hash_id) {
    Opts o;
    memset(&o, 0, sizeof(o));
    o.hash_id = hash_id;
    Air air = fib_air(k, 0, results, o);
    air.asserts.clear();  // rebuilt once n is known from the proof
    int r = verify_fib(proof, len, air);
    return r;
}
// generic AIR (flat description, see parse_air): trace [w][n]
long wfo_prove_air(const uint64_t* desc, size_t desc_len, const uint64_t* trace, size_t n, const uint32_t* opts, uint8_t* out,
                   size_t cap, const uint64_t* tamper, size_t ntamper, uint64_t* positions, size_t* npositions) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return -2;
    air.n = n; air.o = make_opts(opts);
    if (air.aw) return -3;  // multi-segment AIRs go through wfo_prove_air_aux
    return prove_entry(air, trace, nullptr, nullptr, tamper, ntamper, positions, npositions, out, cap);
}
// multi-segment AIR: `builder` fills the aux columns [aw][n][d] from the drawn random elements [nr][d]
long wfo_prove_air_aux(const uint64_t* desc, size_t desc_len, const uint64_t* trace, size_t n, const uint32_t* opts,
                       int (*builder)(void*, const uint64_t*, uint64_t*), void* user, uint8_t* out, size_t cap,
                       const uint64_t* tamper, size_t ntamper, uint64_t* positions, size_t* npositions) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return -2;
    air.n = n; air.o = make_opts(opts);
    return prove_entry(air, trace, builder, user, tamper, ntamper, positions, npositions, out, cap);
}
// same with Air::get_aux_assertions as a callback on the random elements (prover and verifier must be given the same one)
long wfo_prove_air_aux_dyn(const uint64_t* desc, size_t desc_len, const uint64_t* trace, size_t n, const uint32_t* opts,
                           int (*builder)(void*, const uint64_t*, uint64_t*), int (*values_fn)(void*, const uint64_t*, uint64_t*),
                           void* user, uint8_t* out, size_t cap, const uint64_t* tamper, size_t ntamper, uint64_t* positions,
                           size_t* npositions) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return -2;
    air.n = n; air.o = make_opts(opts);
    air.aux_values_fn = values_fn; air.aux_values_user = user;
    return prove_entry(air, trace, builder, user, tamper, ntamper, positions, npositions, out, cap);
}
int wfo_verify_air_dyn(const uint64_t* desc, size_t desc_len, const uint8_t* proof, size_t len, int hash_id,
                       int (*values_fn)(void*, const uint64_t*, uint64_t*), void* user) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return -2;
    memset(&air.o, 0, sizeof(air.o));
    air.o.hash_id = hash_id;
    air.aux_values_fn = values_fn; air.aux_values_user = user;
    return verify_fib(proof, len, air);
}
int wfo_verify_air(const uint64_t* desc, size_t desc_len, const uint8_t* proof, size_t len, int hash_id) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return -2;
    memset(&air.o, 0, sizeof(air.o));
    air.o.hash_id = hash_id;
    return verify_fib(proof, len, air);
}
// Aux columns of the two-segment test AIR tests/airs.py perm_rap (the user's Prover::build_aux_trace for
// that AIR; test helper so that 2^18-row cases do not loop in Python). trace [3][n] (x0, x1, b), rand =
// [gamma, alpha] (d words each), out [3][n][d]:  p' = p (x0 + gamma) / (b + gamma), p[0] = 1;
// q' = q + alpha k x1 p, q[0] = 0, k = 1,2,3,4 periodic;  c[i] = 5 + i.
void wfo_perm_rap_aux(const uint64_t* trace, size_t n, int d, const uint64_t* rand, uint64_t* out) {
    Field F{d};
    EE g = F.zero(), al = F.zero();
    for (int k = 0; k < d; k++) { g.v[k] = rand[k]; al.v[k] = rand[d + k]; }
    EE p = F.one(), q = F.zero();
    for (size_t i = 0; i < n; i++) {
        for (int k = 0; k < d; k++) {
            out[(0 * n + i) * d + k] = p.v[k];
            out[(1 * n + i) * d + k] = q.v[k];
            out[(2 * n + i) * d + k] = k == 0 ? (u64)(5 + i) : 0;
        }
        u64 kk = (u64)(i % 4) + 1;
        q = F.add(q, F.mul(F.mul_base(al, f_mul(kk, trace[n + i])), p));
        EE num = g, den = g;
        num.v[0] = f_add(num.v[0], trace[i]);
        den.v[0] = f_add(den.v[0], trace[2 * n + i]);
        p = F.mul(F.mul(p, num), F.inv(den));
    }
}
// Boundary constraint groups of the main segment as the prover and verifier use them, flattened for the
// known-answer test against air/src/air/tests.rs::get_boundary_constraints:
//   [ngroups, {a, b, nentries, {column, cc (first word), x_offset, poly_len, poly...}*}*]; returns words written
long wfo_boundary_groups(const uint64_t* desc, size_t desc_len, size_t n, const uint64_t* coeffs, uint64_t* out, size_t cap) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return -2;
    air.n = n;
    memset(&air.o, 0, sizeof(air.o));
    air.o.ext = 1;
    std::vector<EE> cc;
    for (size_t i = 0; i < air.asserts.size(); i++) cc.push_back(EE{{coeffs[i], 0, 0}});
    std::vector<u64> w;
    auto groups = boundary_groups(air, cc);
    w.push_back(groups.size());
    for (auto& G : groups) {
        w.push_back(G.a); w.push_back(G.b); w.push_back(G.e.size());
        for (auto& e : G.e) {
            w.push_back(e.col); w.push_back(e.cc.v[0]); w.push_back(e.x_offset); w.push_back(e.poly.size());
            for (auto& c : e.poly) w.push_back(c.v[0]);
        }
    }
    if (w.size() > cap) return -1;
    memcpy(out, w.data(), w.size() * 8);
    return (long)w.size();
}
// The combined, divisor-normalised constraint evaluations the prover computes on CE rows rows[0..k) (step 2 of prove_fib),
// from the frames the caller passes: cur / nxt = [k][w] main LDE rows (i << log2(blowup / ce_blowup) and the row `blowup`
// after it), acur / anxt = [k][aw][ext] aux LDE rows (null without an aux segment). coeffs = [transition main, aux |
// boundary main, aux][ext] as wf_eval_constraints takes them (boundary coefficients in sorted-assertion order), rand =
// [nr][ext]. The periodic and sequence tables are built as the prover builds them. out = [k][ext]. Returns 0, -2 for a
// malformed description, -3 for bad shapes.
long wfo_eval_constraint_rows(const uint64_t* desc, size_t desc_len, size_t n, size_t blowup, int ext, const uint64_t* coeffs,
                              const uint64_t* rand, const uint64_t* rows, size_t k, const uint64_t* cur, const uint64_t* nxt,
                              const uint64_t* acur, const uint64_t* anxt, uint64_t* out) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return -2;
    air.n = n;
    memset(&air.o, 0, sizeof(air.o));
    air.o.ext = (u32)ext; air.o.blowup = (u32)blowup;
    if (ext < 1 || ext > 3 || n < 2 || (n & (n - 1)) || blowup < air.ce_blowup() || (blowup & (blowup - 1)) ||
        (air.aw && (!acur || !anxt)))
        return -3;
    const size_t ce = n * air.ce_blowup();
    for (size_t r = 0; r < k; r++) if (rows[r] >= ce) return -3;
    const size_t ncc = air.num_transition() + air.num_assertions();
    std::vector<EE> cc(ncc), rnd(air.nr);
    for (size_t j = 0; j < ncc; j++) for (int q = 0; q < ext; q++) cc[j].v[q] = coeffs[j * ext + q];
    for (size_t j = 0; j < air.nr; j++) for (int q = 0; q < ext; q++) rnd[j].v[q] = rand[j * ext + q];
    const CeEvaluator ev(air, ext, cc, rnd.data());
    const size_t w = air.width(), aw = air.aw * ext;
    CeEvaluator::Scratch s = ev.scratch();
    for (size_t r = 0; r < k; r++) {
        EE v = ev.row(rows[r], cur + r * w, nxt + r * w, aw ? acur + r * aw : nullptr, aw ? anxt + r * aw : nullptr, s);
        for (int q = 0; q < ext; q++) out[r * ext + q] = v.v[q];
    }
    return 0;
}
// MerkleTree::verify_batch (crypto/src/merkle/mod.rs:300-330) = BatchMerkleProof::get_root + comparison:
// serialized batch proof, the opened leaves (k x 32 bytes, in the order of `indexes`). 0 = accepted.
int wfo_merkle_verify_batch(int hash_id, const uint8_t root[32], const uint64_t* indexes, size_t k, const uint8_t* leaves,
                            const uint8_t* proof, size_t proof_len) {
    Reader r{proof, proof_len};
    BatchProof bp;
    if (!read_batch_proof(r, bp, hash_id) || r.pos != proof_len) return 1;
    std::vector<u64> idx(indexes, indexes + k);
    std::vector<std::array<u8, 32>> lv(k);
    for (size_t i = 0; i < k; i++) memcpy(lv[i].data(), leaves + 32 * i, 32);
    u8 got[32];
    if (!batch_root(hash_id, bp, idx, lv, got)) return 2;
    return memcmp(got, root, 32) ? 3 : 0;
}
// periodic values the evaluator reads at CE step `step` (PeriodicValueTable::get_row, periodic_table.rs:78-82)
long wfo_periodic_row(const uint64_t* desc, size_t desc_len, size_t n, size_t step, uint64_t* out) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return -2;
    air.n = n;
    auto t = periodic_value_table(air);
    for (size_t j = 0; j < t.size(); j++) out[j] = t[j][step % t[j].size()];
    return (long)t.size();
}
size_t wfo_ce_blowup(const uint64_t* desc, size_t desc_len) {
    Air air;
    if (!parse_air(desc, desc_len, air)) return 0;
    return air.ce_blowup();
}
// ByteWriter::write_usize (utils/core/src/serde/byte_writer.rs:77-92): vint64; returns the encoded length
size_t wfo_write_usize(uint64_t value, uint8_t out[9]) {
    std::vector<u8> b;
    write_vint64(b, value);
    memcpy(out, b.data(), b.size());
    return b.size();
}
// Context::to_elements (air/src/proof/context.rs:119-136) for arbitrary parameters; returns the count
size_t wfo_context_elements(size_t main_width, size_t aux_width, size_t aux_rands, size_t trace_length, size_t num_constraints,
                            const uint32_t* opts, uint64_t* out) {
    Air a;
    a.w = main_width; a.aw = aux_width; a.nr = aux_rands; a.n = trace_length; a.o = make_opts(opts);
    // num_constraints is carried by the (assertions + transition) count of the description
    a.degrees.assign(num_constraints, {1, {}});
    std::vector<u64> e = context_elements(a);
    memcpy(out, e.data(), e.size() * 8);
    return e.size();
}
// PartitionOptions::partition_size / num_partitions (air/src/options.rs:428-444)
size_t wfo_partition_size(size_t num_partitions, size_t hash_rate, size_t ext_degree, size_t num_columns) {
    if (num_partitions == 1) return num_columns;
    size_t min_partition_size = hash_rate / ext_degree;
    return std::max((num_columns + num_partitions - 1) / num_partitions, min_partition_size);
}
size_t wfo_num_partitions(size_t num_partitions, size_t hash_rate, size_t ext_degree, size_t num_columns) {
    size_t ps = wfo_partition_size(num_partitions, hash_rate, ext_degree, num_columns);
    return (num_columns + ps - 1) / ps;
}
// builds the FibSmall x k trace: pair j starts at (j+1, j+1); results[j] = last value of column 2j+1
void wfo_build_fib_trace(size_t k, size_t n, uint64_t* trace, uint64_t* results) {
    for (size_t j = 0; j < k; j++) {
        u64 a = j + 1, b2 = j + 1;
        for (size_t i = 0; i < n; i++) {
            trace[(2 * j) * n + i] = a; trace[(2 * j + 1) * n + i] = b2;
            a = f_add(a, b2); b2 = f_add(b2, a);  // examples/src/fibonacci/fib_small/prover.rs build_trace
        }
        results[j] = trace[(2 * j + 1) * n + n - 1];
    }
}
}
