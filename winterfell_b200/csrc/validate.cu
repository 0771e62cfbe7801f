// validate.cu — the reference's debug-build checks of a trace against its AIR, on the device:
//   * Trace::validate (prover/src/trace/mod.rs:86-201): every main and aux assertion, then every transition constraint on
//     steps 0 .. n - exemptions over the trace-domain evaluations (assertion_check_kernel, transition_check_kernel);
//   * ConstraintEvaluationTable::validate_transition_degrees (prover/src/constraints/evaluation_table.rs:181-230, 421-477):
//     each transition constraint's evaluations over the CE domain divided by the transition divisor (transition_columns_kernel),
//     one batched plain inverse NTT of the CE x (n_mtr + n_atr * D) matrix, the highest non-zero coefficient per column
//     (degree_kernel), compared with the declared degrees.
// The programs run on the interpreter of constraints_generic.cuh (run_main_program / run_aux_program).
#include <cstdarg>

#include "air_host.hpp"
#include "constraints_generic.cuh"

namespace {

// Registers of CE row (or trace step) i as generic_constraints_row loads them: frame rows i << (log_blowup - log_ce_blowup)
// and the row 2^log_blowup further (wrapping), periodic values, then (AUX) everything in E with the random elements. With a
// row window (p.ce_rows != 0, as in the constraint kernels) the matrices hold the rows of CE rows [p.row0, p.row0 + ce_rows)
// followed by the next-state rows, so the loads are local and do not wrap; periodic values stay keyed on the global row i.
template <int D, bool AUX>
__device__ __forceinline__ void load_registers(const GenEvalParams& p, size_t i, u64* r, GlExt<D>* ra) {
    const size_t N = (size_t)1 << (p.log_n + p.log_blowup);
    const size_t ls = (i - p.row0) << (p.log_blowup - p.log_ce_blowup);
    const size_t nx = p.ce_rows ? ls + ((size_t)1 << p.log_blowup) : ((ls + ((size_t)1 << p.log_blowup)) & (N - 1));
    for (u32 c = 0; c < p.w; c++) { r[c] = seg_at(p.lde, ls, c); r[p.w + c] = seg_at(p.lde, nx, c); }
    for (u32 j = 0; j < p.num_periodic; j++) r[2 * p.w + j] = p.ptab[p.ptab_off[j] + (u32)(i & (p.ptab_len[j] - 1))];
    if constexpr (AUX) {
        for (u32 c = 0; c < 2 * p.w; c++) ra[c] = ext_from_base<D>(r[c]);
        for (u32 j = 0; j < p.aw; j++) {
#pragma unroll
            for (int q = 0; q < D; q++) {
                ra[2 * p.w + j].v[q] = seg_at(p.alde, ls, j * D + q);
                ra[2 * p.w + p.aw + j].v[q] = seg_at(p.alde, nx, j * D + q);
            }
        }
        const u32 pb = 2 * p.w + 2 * p.aw;
        for (u32 j = 0; j < p.num_periodic; j++) ra[pb + j] = ext_from_base<D>(r[2 * p.w + j]);
        for (u32 j = 0; j < p.nr; j++) ra[pb + p.num_periodic + j] = ld_ext<D>(p.rnd + (size_t)j * D);
    }
}

// Per transition step i in [step0, step0 + steps): constraint j fails when the sum of its OUT values is non-zero. Constraints
// with one OUT are tested as it runs; those with several (slot[j] != ~0) are summed in this step's row of `acc` (zeroed,
// [steps][slots][D]) and tested after the program. first[j] (main, then aux) = the smallest failing step.
struct TransitionCheck {
    GenEvalParams g;
    size_t step0, steps;
    const u32 *mslot, *aslot;   // [n_mtr], [n_atr]
    u32 nmslots, naslots;
    u64 *macc, *aacc;
    const u32 *mslot_con, *aslot_con;  // slot -> constraint
    u32 n_mtr;
    unsigned long long* first;
};

template <int D, bool AUX>
__global__ void __launch_bounds__(128) transition_check_kernel(TransitionCheck c) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= c.steps) return;
    const size_t i = c.step0 + t;
    const GenEvalParams& p = c.g;
    u64 r[GEN_MAX_REGS];
    GlExt<D> ra[AUX ? AUX_MAX_REGS : 1];
    load_registers<D, AUX>(p, i, r, ra);
    u64* macc = c.macc + t * c.nmslots;
    u64* aacc = c.aacc + t * c.naslots * D;
    run_main_program(p, r, [&](u32 j, u64 v) {
        const u32 s = c.mslot[j];
        if (s == ~0u) { if (v) atomicMin(&c.first[j], (unsigned long long)i); }
        else macc[s] = gl_add(macc[s], v);
    });
    for (u32 s = 0; s < c.nmslots; s++) if (macc[s]) atomicMin(&c.first[c.mslot_con[s]], (unsigned long long)i);
    if constexpr (AUX) {
        run_aux_program<D>(p, ra, [&](u32 j, const GlExt<D>& v) {
            const u32 s = c.aslot[j];
            if (s == ~0u) {
                u64 nz = 0;
#pragma unroll
                for (int q = 0; q < D; q++) nz |= v.v[q];
                if (nz) atomicMin(&c.first[c.n_mtr + j], (unsigned long long)i);
            } else {
#pragma unroll
                for (int q = 0; q < D; q++) aacc[s * D + q] = gl_add(aacc[s * D + q], v.v[q]);
            }
        });
        for (u32 s = 0; s < c.naslots; s++) {
            u64 nz = 0;
            for (int q = 0; q < D; q++) nz |= aacc[s * D + q];
            if (nz) atomicMin(&c.first[c.n_mtr + c.aslot_con[s]], (unsigned long long)i);
        }
    }
}

// One thread per asserted cell of one segment. Assertion a covers cells [coff[a], coff[a + 1]): cell k at step
// first_step + k * stride, value vals[voff[a] + (one value ? 0 : k) * D ..]. *res = min over failing cells of (a << 40 | k),
// the reference's order (assertions in description order, each one's steps increasing).
struct AssertionCheck {
    SegMatrix m;
    u32 D, na;
    const u64* coff;   // [na + 1]
    const u64 *col, *first_step, *stride, *voff, *nvals;
    const u64* vals;
    unsigned long long* res;
};
__global__ void __launch_bounds__(256) assertion_check_kernel(AssertionCheck c) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= c.coff[c.na]) return;
    u32 lo = 0, hi = c.na;   // last a with coff[a] <= t
    while (hi - lo > 1) { const u32 mid = (lo + hi) / 2; if (c.coff[mid] <= t) lo = mid; else hi = mid; }
    const u32 a = lo;
    const u64 k = t - c.coff[a];
    const size_t step = c.first_step[a] + k * c.stride[a];
    const u64* v = c.vals + c.voff[a] + (c.nvals[a] == 1 ? 0 : k * c.D);
    u64 diff = 0;
    for (u32 q = 0; q < c.D; q++) diff |= seg_at(c.m, step, (u32)c.col[a] * c.D + q) ^ v[q];
    if (diff) atomicMin(c.res, ((unsigned long long)a << 40) | k);
}

// Per CE row i: constraint j's raw evaluation times prod_k (x - g^(n-k)) / (x^n - 1), x = 7 w_ce^i, into column j (main) or
// columns n_mtr + j*D + q (aux) of `out` (zeroed: several OUTs of one constraint add up). With a row window (p.ce_rows != 0)
// the launch covers CE rows [p.row0, p.row0 + ce_rows) and row i goes to row i - row0 of `out`.
template <int D, bool AUX>
__global__ void __launch_bounds__(128) transition_columns_kernel(GenEvalParams p, u32 n_mtr) {
    const size_t ce = (size_t)1 << (p.log_n + p.log_ce_blowup);
    const size_t il = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (il >= (p.ce_rows ? p.ce_rows : ce)) return;
    const size_t i = p.row0 + il;
    const u32 half = (u32)(ce >> 1);
    u64 w = p.tw_ce[i & (half - 1)];
    if (i & half) w = gl_neg(w);
    const u64 x = gl_mul(w, GL_GENERATOR);
    u64 f = p.zt[i & (((size_t)1 << p.log_ce_blowup) - 1)];
    for (u32 k = 0; k < p.num_exempt; k++) f = gl_mul(f, gl_sub(x, p.exempt[k]));
    u64 r[GEN_MAX_REGS];
    GlExt<D> ra[AUX ? AUX_MAX_REGS : 1];
    load_registers<D, AUX>(p, i, r, ra);
    auto cell = [&](u32 col) -> u64& { return p.out.base[(size_t)(col / p.out.W) * p.out.seg_stride + il * p.out.W + (col % p.out.W)]; };
    run_main_program(p, r, [&](u32 j, u64 v) { u64& d = cell(j); d = gl_add(d, gl_mul(v, f)); });
    if constexpr (AUX) {
        run_aux_program<D>(p, ra, [&](u32 j, const GlExt<D>& v) {
#pragma unroll
            for (int q = 0; q < D; q++) { u64& d = cell(n_mtr + j * D + q); d = gl_add(d, gl_mul(v.v[q], f)); }
        });
    }
}

// deg1[col] = 1 + the highest row of column col that is non-zero (0: the zero polynomial). Grid: (row blocks, columns).
__global__ void __launch_bounds__(256) degree_kernel(SegMatrix m, unsigned long long* deg1) {
    const u32 col = blockIdx.y;
    unsigned long long best = 0;
    for (size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x; row < m.rows; row += (size_t)gridDim.x * blockDim.x)
        if (seg_at(m, row, col)) best = row + 1;   // rows increase along the loop
#pragma unroll
    for (int o = 16; o; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o); best = t > best ? t : best; }
    if ((threadIdx.x & 31) == 0 && best) atomicMax(&deg1[col], best);
}

// host-side uploads of one check: stream-ordered copies from vectors that live until the check's synchronisation
struct Uploads {
    DevScratch dev;
    std::vector<std::vector<u64>> keep;
    explicit Uploads(wf_ctx* c) : dev(c) {}
    template <class T>
    int put(const std::vector<T>& v, const T** out) {
        void* p;
        const size_t bytes = v.size() * sizeof(T);
        CKI(dev.alloc(std::max(bytes, (size_t)8), &p));
        wf_ctx* ctx = dev.ctx;
        if (bytes) CK(cudaMemcpyAsync(p, v.data(), bytes, cudaMemcpyHostToDevice, ctx->st));
        *out = (const T*)p;
        return WF_OK;
    }
};

std::string fmt(const char* f, ...) {
    char b[512];
    va_list ap;
    va_start(ap, f);
    vsnprintf(b, sizeof(b), f, ap);
    va_end(ap);
    return b;
}

// the fields of GenEvalParams both checks share: programs, constants, registers and the aux segment
int program_params(Uploads& up, const AirHost& air, const wf_mat* main, const wf_mat* aux, const u64* rnd, int D, GenEvalParams& p) {
    memset(&p, 0, sizeof(p));
    p.lde = main->m; p.w = air.w;
    p.prog_len = (u32)(air.prog.size() / 4); p.num_regs = air.num_regs; p.num_periodic = (u32)air.periodic.size();
    p.num_tc = (u32)air.degrees.size();
    CKI(up.put(air.prog, &p.prog));
    CKI(up.put(air.consts, &p.consts));
    if (aux) {
        p.alde = aux->m; p.aw = air.aw; p.nr = air.nr; p.aprog_len = (u32)(air.aux_prog.size() / 4);
        CKI(up.put(air.aux_prog, &p.aprog));
        CKI(up.put(std::vector<u64>(rnd, rnd + (size_t)air.nr * D), &p.rnd));
    }
    return WF_OK;
}

// OUT instructions per constraint -> slot of every constraint with more than one (~0: one or none), and slot -> constraint
void out_slots(const std::vector<u32>& prog, size_t ncon, std::vector<u32>& slot, std::vector<u32>& slot_con) {
    std::vector<u32> cnt(ncon, 0);
    for (size_t k = 0; k < prog.size(); k += 4) if (prog[k] == 4) cnt[prog[k + 1]]++;
    slot.assign(ncon, ~0u);
    for (size_t j = 0; j < ncon; j++) if (cnt[j] > 1) { slot[j] = (u32)slot_con.size(); slot_con.push_back((u32)j); }
    if (slot_con.empty()) slot_con.push_back(0);   // a non-empty upload
}

std::string elem_str(const u64* v, int D) {
    if (D == 1) return fmt("%llu", (unsigned long long)v[0]);
    std::string s = "(";
    for (int q = 0; q < D; q++) s += fmt(q ? ", %llu" : "%llu", (unsigned long long)v[q]);
    return s + ")";
}

template <int D>
int check_trace_part(wf_ctx* ctx, const AirHost& air, const TraceCheckPart& w, const u64* rnd, u32 log_n, std::vector<u64>& raw) {
    const size_t n = (size_t)1 << log_n;
    const wf_mat *main = w.main, *aux = w.aux;
    const u32 n_mtr = (u32)air.degrees.size(), n_atr = aux ? (u32)air.aux_degrees.size() : 0, n_tr = n_mtr + n_atr;
    Uploads up(ctx);
    GenEvalParams p;
    CKI(program_params(up, air, main, aux, rnd, D, p));
    p.log_n = log_n;   // log_blowup = log_ce_blowup = 0: the frame is rows (i, i + 1) of the trace
    p.row0 = w.row0; p.ce_rows = w.rows;
    // periodic value j at step i is col_j[i mod L_j]: the periodic polynomial at g^(i n / L_j)
    std::vector<u64> ptab;
    std::vector<u32> poff, plen;
    for (auto& col : air.periodic) { poff.push_back((u32)ptab.size()); plen.push_back((u32)col.size()); ptab.insert(ptab.end(), col.begin(), col.end()); }
    CKI(up.put(ptab, &p.ptab));
    CKI(up.put(poff, &p.ptab_off));
    CKI(up.put(plen, &p.ptab_len));
    // results: [0] main assertions, [1] aux assertions, [2..] first failing step per transition constraint
    void* d_res;
    CKI(up.dev.alloc((2 + (size_t)n_tr) * 8, &d_res));
    CK(cudaMemsetAsync(d_res, 0xFF, (2 + (size_t)n_tr) * 8, ctx->st));
    unsigned long long* res = (unsigned long long*)d_res;
    // assertions: main in description order, then aux (values in E: the first D of each value's three words). A main
    // assertion on a column outside [acol0, acol0 + amain.cols) keeps its index and gets no cells.
    for (int seg = 0; seg < (aux ? 2 : 1); seg++) {
        const auto& as = seg ? air.aux_asserts : air.asserts;
        const u32 wpv = seg ? 3 : 1, d = seg ? D : 1;
        std::vector<u64> coff = {0}, col, fs, st, voff, nv, vals;
        for (auto& a : as) {
            const bool mine = seg || (a.column >= w.acol0 && a.column < w.acol0 + w.amain.cols);
            const size_t k = a.values.size() / wpv;
            col.push_back(seg ? a.column : a.column - w.acol0); fs.push_back(a.first_step); st.push_back(a.stride); nv.push_back(k);
            voff.push_back(vals.size());
            for (size_t i = 0; i < k; i++) for (u32 q = 0; q < d; q++) vals.push_back(a.values[i * wpv + q]);
            coff.push_back(coff.back() + (!mine ? 0 : a.stride ? n / a.stride : 1));
        }
        if (coff.back() == 0) continue;
        AssertionCheck c;
        c.m = !seg ? w.amain : w.aasrt.base ? w.aasrt : aux->m; c.D = d; c.na = (u32)as.size(); c.res = res + seg;
        CKI(up.put(coff, &c.coff)); CKI(up.put(col, &c.col)); CKI(up.put(fs, &c.first_step)); CKI(up.put(st, &c.stride));
        CKI(up.put(voff, &c.voff)); CKI(up.put(nv, &c.nvals)); CKI(up.put(vals, &c.vals));
        assertion_check_kernel<<<(unsigned)((coff.back() + 255) / 256), 256, 0, ctx->st>>>(c);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    // transitions on steps [s0, s1)
    TransitionCheck t;
    t.g = p; t.step0 = w.s0; t.steps = w.s1 > w.s0 ? w.s1 - w.s0 : 0; t.n_mtr = n_mtr; t.first = res + 2;
    std::vector<u32> ms, msc, as_, asc;
    out_slots(air.prog, n_mtr, ms, msc);
    out_slots(aux ? air.aux_prog : std::vector<u32>(), n_atr, as_, asc);
    t.nmslots = (u32)std::count_if(ms.begin(), ms.end(), [](u32 s) { return s != ~0u; });
    t.naslots = (u32)std::count_if(as_.begin(), as_.end(), [](u32 s) { return s != ~0u; });
    CKI(up.put(ms, &t.mslot)); CKI(up.put(msc, &t.mslot_con)); CKI(up.put(as_, &t.aslot)); CKI(up.put(asc, &t.aslot_con));
    void* acc;
    const size_t acc_words = t.steps * (t.nmslots + (size_t)t.naslots * D);
    CKI(up.dev.alloc(std::max(acc_words, (size_t)1) * 8, &acc));
    if (acc_words) CK(cudaMemsetAsync(acc, 0, acc_words * 8, ctx->st));
    t.macc = (u64*)acc; t.aacc = (u64*)acc + t.steps * t.nmslots;
    if (t.steps) {
        const unsigned blocks = (unsigned)((t.steps + 127) / 128);
        if (aux) transition_check_kernel<D, true><<<blocks, 128, 0, ctx->st>>>(t);
        else transition_check_kernel<D, false><<<blocks, 128, 0, ctx->st>>>(t);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    raw.assign(2 + (size_t)n_tr, 0);
    CK(cudaMemcpyAsync(raw.data(), d_res, raw.size() * 8, cudaMemcpyDeviceToHost, ctx->st));
    CK(cudaStreamSynchronize(ctx->st));
    return WF_OK;
}

template <int D>
int transition_columns(wf_ctx* ctx, const AirHost& air, const wf_mat* lde, const wf_mat* alde, const u64* rnd, u32 log_n, u32 log_b,
                       size_t row0, size_t ce_rows, const SegMatrix& out) {
    const size_t n = (size_t)1 << log_n;
    const u32 log_ceb = air.log_ce_blowup();
    const size_t ce = n << log_ceb;
    const u32 n_mtr = (u32)air.degrees.size();
    Uploads up(ctx);
    GenEvalParams p;
    CKI(program_params(up, air, lde, alde, rnd, D, p));
    p.log_n = log_n; p.log_blowup = log_b; p.log_ce_blowup = log_ceb;
    p.row0 = row0; p.ce_rows = ce_rows;
    std::vector<u64> ptab;
    std::vector<u32> poff, plen;
    air.periodic_ce_tables(n, log_ceb, ptab, poff, plen);
    CKI(up.put(ptab, &p.ptab));
    CKI(up.put(poff, &p.ptab_off));
    CKI(up.put(plen, &p.ptab_len));
    CKI(wf_get_twiddles(ctx, log_n + log_ceb, &p.tw_ce));
    std::vector<u64> zt((size_t)1 << log_ceb);   // 1 / (x^n - 1) at CE row i mod ce_blowup, as eval_constraints builds it
    const u64 o_n = gl_pow(GL_GENERATOR, n), w_ceb = gl_root_of_unity(log_ceb);
    for (u32 i = 0; i < (1u << log_ceb); i++) zt[i] = gl_inv(gl_sub(gl_mul(o_n, gl_pow(w_ceb, i)), 1));
    CKI(up.put(zt, &p.zt));
    const u64 g_tr = gl_root_of_unity(log_n);
    p.num_exempt = air.exemptions;
    for (u32 e = 0; e < air.exemptions; e++) p.exempt[e] = gl_pow(g_tr, n - air.exemptions + e);  // divisor.rs:31-41
    CK(cudaMemsetAsync(out.base, 0, out.words() * 8, ctx->st));
    p.out = out;
    const unsigned blocks = (unsigned)(((ce_rows ? ce_rows : ce) + 127) / 128);
    if (alde) transition_columns_kernel<D, true><<<blocks, 128, 0, ctx->st>>>(p, n_mtr);
    else transition_columns_kernel<D, false><<<blocks, 128, 0, ctx->st>>>(p, n_mtr);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(ctx->st));   // the uploads' host vectors end with this scope
    return WF_OK;
}

}  // namespace

int wf_check_trace_part(wf_ctx* ctx, const AirHost& air, const TraceCheckPart& part, const u64* rnd, u32 log_n, int D, std::vector<u64>& raw) {
    switch (D) {
        case 1: return check_trace_part<1>(ctx, air, part, rnd, log_n, raw);
        case 2: return check_trace_part<2>(ctx, air, part, rnd, log_n, raw);
        case 3: return check_trace_part<3>(ctx, air, part, rnd, log_n, raw);
    }
    return wf_fail(ctx, WF_ERR_UNSUPPORTED, "field extension %d", D);
}

void wf_trace_verdict(const AirHost& air, bool aux, int D, const std::vector<u64>& h, TraceReport& rep) {
    const u32 n_mtr = (u32)air.degrees.size(), n_tr = n_mtr + (aux ? (u32)air.aux_degrees.size() : 0);
    rep.first_fail.assign(h.begin() + 2, h.begin() + 2 + n_tr);
    // the first violation the reference panics on: main assertions, aux assertions, then the smallest failing step with main
    // constraints before aux ones
    for (int seg = 0; seg < 2; seg++) {
        if (h[seg] == ~0ull) continue;
        const auto& a = (seg ? air.aux_asserts : air.asserts)[h[seg] >> 40];
        const u64 k = h[seg] & ((1ull << 40) - 1);
        rep.kind = seg ? WF_VIOLATION_AUX_ASSERTION : WF_VIOLATION_MAIN_ASSERTION;
        rep.index = (u32)(h[seg] >> 40); rep.column = (u32)a.column; rep.step = a.first_step + k * a.stride;
        const size_t vi = a.values.size() / (seg ? 3 : 1) == 1 ? 0 : k;
        rep.msg = fmt("trace does not satisfy assertion %s(%u, %llu) == %s", seg ? "aux_trace" : "main_trace", rep.column,
                      (unsigned long long)rep.step, elem_str(&a.values[vi * (seg ? 3 : 1)], seg ? D : 1).c_str());
        return;
    }
    u64 best = ~0ull;
    u32 bj = 0;
    for (u32 j = 0; j < n_tr; j++) if (rep.first_fail[j] < best) { best = rep.first_fail[j]; bj = j; }
    if (best != ~0ull) {
        const bool main_seg = bj < n_mtr;
        rep.kind = main_seg ? WF_VIOLATION_MAIN_TRANSITION : WF_VIOLATION_AUX_TRANSITION;
        rep.index = main_seg ? bj : bj - n_mtr; rep.step = best; rep.column = 0;
        rep.msg = fmt("%s transition constraint %u did not evaluate to ZERO at step %llu", main_seg ? "main" : "auxiliary", rep.index,
                      (unsigned long long)best);
    }
}

int wf_check_trace(wf_ctx* ctx, const AirHost& air, const wf_mat* main, const wf_mat* aux, const u64* rnd, u32 log_n, int D,
                   TraceReport& rep) {
    TraceCheckPart part;
    part.amain = main->m; part.main = main; part.aux = aux;
    part.s1 = ((size_t)1 << log_n) - air.exemptions;
    std::vector<u64> raw;
    CKI(wf_check_trace_part(ctx, air, part, rnd, log_n, D, raw));
    wf_trace_verdict(air, aux != nullptr, D, raw, rep);
    return WF_OK;
}

int wf_transition_columns(wf_ctx* ctx, const AirHost& air, const wf_mat* lde, const wf_mat* alde, const u64* rnd, u32 log_n, u32 log_b,
                          int D, size_t row0, size_t ce_rows, const SegMatrix& out) {
    switch (D) {
        case 1: return transition_columns<1>(ctx, air, lde, alde, rnd, log_n, log_b, row0, ce_rows, out);
        case 2: return transition_columns<2>(ctx, air, lde, alde, rnd, log_n, log_b, row0, ce_rows, out);
        case 3: return transition_columns<3>(ctx, air, lde, alde, rnd, log_n, log_b, row0, ce_rows, out);
    }
    return wf_fail(ctx, WF_ERR_UNSUPPORTED, "field extension %d", D);
}

int wf_column_degrees(wf_ctx* ctx, wf_mat*& cols, std::vector<u64>& deg1) {
    // coefficients by a plain inverse NTT, as the reference: the domain offset scales coefficient k by 7^-k and moves no zero
    wf_mat* coefs = nullptr;
    struct Free { wf_ctx* c; wf_mat** a; ~Free() { wf_mat_free(c, *a); } } fr{ctx, &coefs};
    const size_t ce = cols->m.rows;
    const u32 ncols = cols->m.cols;
    CKI(wf_mat_interpolate(ctx, cols, &coefs));
    wf_mat_free(ctx, cols);
    cols = nullptr;
    DevScratch dev(ctx);
    void* d_deg;
    CKI(dev.alloc((size_t)ncols * 8, &d_deg));
    CK(cudaMemsetAsync(d_deg, 0, (size_t)ncols * 8, ctx->st));
    const unsigned rb = (unsigned)std::min<size_t>((ce + 255) / 256, 1024);
    degree_kernel<<<dim3(rb, ncols), 256, 0, ctx->st>>>(coefs->m, (unsigned long long*)d_deg);
    ctx->launches++;
    CK(cudaGetLastError());
    deg1.assign(ncols, 0);
    CK(cudaMemcpyAsync(deg1.data(), d_deg, ncols * 8, cudaMemcpyDeviceToHost, ctx->st));
    CK(cudaStreamSynchronize(ctx->st));
    return WF_OK;
}

void wf_degree_verdict(const AirHost& air, bool aux, int D, u32 log_n, const std::vector<u64>& deg1, TraceReport& rep) {
    const size_t n = (size_t)1 << log_n, ce = n << air.log_ce_blowup();
    const u32 n_mtr = (u32)air.degrees.size(), n_tr = n_mtr + (aux ? (u32)air.aux_degrees.size() : 0);
    // expected: get_evaluation_degree(n) - (n - exemptions) (transition/degree.rs:90-96, evaluation_table.rs:421-437)
    auto degs = air.all_degrees();
    rep.expected.assign(n_tr, 0);
    rep.actual.assign(n_tr, 0);
    u64 max_deg = 0;
    for (u32 j = 0; j < n_tr; j++) {
        u64 e = (u64)degs[j].first * (n - 1);
        for (u32 cyc : degs[j].second) e += (n / cyc) * (cyc - 1);
        rep.expected[j] = e - (n - air.exemptions);
        u64 d1 = 0;
        if (j < n_mtr) d1 = deg1[j];
        else for (int q = 0; q < D; q++) d1 = std::max(d1, deg1[n_mtr + (j - n_mtr) * D + q]);
        rep.actual[j] = d1 ? d1 - 1 : 0;   // polynom::degree_of
        max_deg = std::max(max_deg, rep.actual[j]);
    }
    if (rep.kind != WF_VALID) return;
    if (rep.expected != rep.actual) {
        auto list = [](const std::vector<u64>& v) {
            std::string s = "[";
            for (size_t i = 0; i < v.size(); i++) s += fmt(i ? ", %3llu" : "%3llu", (unsigned long long)v[i]);
            return s + "]";
        };
        rep.kind = WF_VIOLATION_DEGREES;
        rep.msg = "transition constraint degrees didn't match\nexpected: " + list(rep.expected) + "\nactual:   " + list(rep.actual);
        return;
    }
    u64 dom = 1;
    while (dom < std::max<u64>(max_deg, n + 1)) dom <<= 1;
    if (dom != ce) {
        rep.kind = WF_VIOLATION_CE_DOMAIN;
        rep.msg = fmt("incorrect constraint evaluation domain size; expected %llu, but was %llu", (unsigned long long)dom, (unsigned long long)ce);
    }
}

int wf_check_degrees(wf_ctx* ctx, const AirHost& air, const wf_mat* lde, const wf_mat* alde, const u64* rnd, u32 log_n, u32 log_b,
                     int D, TraceReport& rep) {
    const u32 log_ceb = air.log_ce_blowup();
    const u32 ncols = (u32)air.degrees.size() + (alde ? (u32)air.aux_degrees.size() * D : 0);
    if (log_ceb > log_b) return wf_fail(ctx, WF_ERR_INVALID, "blowup factor too small for the constraint degrees");
    // CE x ncols transition evaluations over the divisor, then the degree of every column
    wf_mat* cols = nullptr;
    CKI(wf_mat_alloc(ctx, (size_t)1 << (log_n + log_ceb), ncols, &cols));
    struct Free { wf_ctx* c; wf_mat** a; ~Free() { wf_mat_free(c, *a); } } fr{ctx, &cols};
    CKI(wf_transition_columns(ctx, air, lde, alde, rnd, log_n, log_b, D, 0, 0, cols->m));
    std::vector<u64> deg1;
    CKI(wf_column_degrees(ctx, cols, deg1));
    wf_degree_verdict(air, alde != nullptr, D, log_n, deg1, rep);
    return WF_OK;
}

extern "C" int wf_ctx_set_validation(wf_ctx* ctx, int on) {
    if (!ctx) return WF_ERR_INVALID;
    ctx->validate = on != 0;
    return WF_OK;
}
