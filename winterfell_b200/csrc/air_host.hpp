// air_host.hpp — the host-side form of an AIR description, shared by the prover (prover.cu) and the trace checks
// (validate.cu).
#pragma once
#include "internal.hpp"

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
        for (auto& dg : all_degrees()) {
            u32 bound = dg.first + (u32)dg.second.size() - 1, l = 0;
            while ((1u << l) < bound) l++;
            r = std::max(r, std::max(l, 1u));
        }
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
