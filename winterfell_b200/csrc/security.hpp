// security.hpp — the reference's security estimator (air/src/proof/security.rs:20-306) for the Goldilocks field:
// ConjecturedSecurity::compute, ProvenSecurity::compute and their is_at_least rules, on the host.
//
// The estimate is an integer made from doubles, so it is restated operation by operation: the same libm calls (log2, pow,
// sqrt, ceil; Rust's f64 methods call the same C library functions) in the same order, f64::min's NaN rule (fmin), the
// saturating float-to-integer casts of Rust's `as` (NaN and negatives to 0) and max_by_key's choice of the LAST maximum.
// A batching factor of 0 (Algebraic / Horner batching of exactly one item) gives log2(0) = -inf and an epsilon of +inf, as
// in the reference. This header relies on IEEE infinities: it must not be compiled with -ffast-math (nvcc's
// --use_fast_math touches device code only).
#pragma once
#include <cmath>
#include <cstdint>
#include <map>
#include <tuple>

#include "air_host.hpp"

namespace wf_security {

constexpr uint32_t BASE_FIELD_BITS = 64;              // Goldilocks
constexpr uint32_t GRINDING_CONTRIBUTION_FLOOR = 80;
constexpr uint64_t MAX_PROXIMITY_PARAMETER = 1000;
constexpr uint32_t BATCH_LINEAR = 0;                  // BatchingMethod::Linear (air/src/options.rs:479-483)

// Hasher::COLLISION_RESISTANCE (crypto/src/hash/blake/mod.rs:27,79; rescue/rp64_256/mod.rs:121; rp64_256_jive/mod.rs:117;
// sha/mod.rs:24); 0 for an unknown hash
static inline uint32_t collision_resistance(int hash_id) {
    switch (hash_id) {
        case WF_HASH_BLAKE3_256: case WF_HASH_RP64_256: case WF_HASH_RPJIVE64_256: case WF_HASH_SHA3_256: return 128;
        case WF_HASH_BLAKE3_192: return 96;
        default: return 0;
    }
}

// `x as u64` / `x as u32`: NaN and everything up to 0 give 0, everything at or above 2^64 (2^32) the maximum
static inline uint64_t sat_u64(double x) {
    if (!(x > 0.0)) return 0;
    if (x >= 18446744073709551616.0) return UINT64_MAX;
    return (uint64_t)x;
}
static inline uint32_t sat_u32(double x) {
    if (!(x > 0.0)) return 0;
    if (x >= 4294967296.0) return UINT32_MAX;
    return (uint32_t)x;
}

// ConjecturedSecurity::compute (security.rs:30-47)
static inline uint32_t conjectured(const Options& o, uint32_t collision_res) {
    const uint32_t field_security = BASE_FIELD_BITS * o.ext;
    uint32_t query_security = (31 - (uint32_t)__builtin_clz(o.blowup)) * o.num_queries;   // blowup_factor().ilog2()
    if (query_security >= GRINDING_CONTRIBUTION_FLOOR) query_security += o.grinding;
    return std::min(std::min(field_security, query_security) - 1, collision_res);
}

static inline double batching_factor(uint32_t method, uint64_t count) {
    return method == BATCH_LINEAR ? 1.0 : (double)count - 1.0;
}

// FriOptions::num_fri_layers (fri/src/options.rs:85-93) of the LDE domain
static inline uint64_t num_fri_layers(const Options& o, uint64_t domain) {
    uint64_t n = 0;
    const uint64_t max_rem = ((uint64_t)o.rem_max_deg + 1) * o.blowup;
    while (domain > max_rem) { domain /= o.folding; n++; }
    return n;
}

// proven_security_protocol_unique_decoding (security.rs:223-285)
static inline uint64_t proven_udr_uncapped(const Options& o, uint64_t trace_length, uint64_t num_constraints, uint64_t num_committed) {
    const double ext_bits = (double)(BASE_FIELD_BITS * o.ext);
    const double q = (double)o.num_queries;
    const uint64_t lde_n = trace_length * o.blowup;
    const double lde = (double)lde_n;
    const double h = (double)trace_length;
    const double num_openings = 2.0;
    const double rho_plus = (h + num_openings) / lde;
    const double alpha = (1.0 + rho_plus) * 0.5;
    const double max_deg = (double)o.blowup + 1.0;
    double acc = INFINITY;
    acc = std::fmin(acc, -std::log2(batching_factor(o.batch_c, num_constraints)) + ext_bits);
    acc = std::fmin(acc, -std::log2(max_deg * (h + num_openings - 1.0) + (h - 1.0)) + ext_bits);
    acc = std::fmin(acc, ext_bits - std::log2(lde * batching_factor(o.batch_d, num_committed)));
    const double folding = (double)o.folding;
    double layers = INFINITY;
    for (uint64_t i = 0, nl = num_fri_layers(o, lde_n); i < nl; i++)
        layers = std::fmin(layers, ext_bits - std::log2((folding - 1.0) * (lde + 1.0)));
    acc = std::fmin(acc, layers);
    acc = std::fmin(acc, (double)o.grinding - std::log2(std::pow(alpha, q)));
    return sat_u64(acc);
}

// proven_security_protocol_for_given_proximity_parameter (security.rs:150-220)
static inline uint64_t proven_ldr_at(const Options& o, uint64_t trace_length, uint32_t m_int, uint64_t num_constraints,
                                     uint64_t num_committed) {
    const double ext_bits = (double)(BASE_FIELD_BITS * o.ext);
    const double q = (double)o.num_queries;
    const double m = (double)m_int;
    const double rho = 1.0 / (double)o.blowup;
    const double alpha = (1.0 + 0.5 / m) * std::sqrt(rho);
    const double max_deg = (double)o.blowup + 1.0;
    const double lde = (double)(trace_length * o.blowup);
    const double h = (double)trace_length;
    const double num_openings = 2.0;
    const double l = m / (rho - (2.0 * m / lde));   // list size; +inf at m = trace_length / 2
    double acc = INFINITY;
    acc = std::fmin(acc, -std::log2(l) - std::log2(batching_factor(o.batch_c, num_constraints)) + ext_bits);
    acc = std::fmin(acc, -std::log2(l * l * (max_deg * (h + num_openings - 1.0) + (h - 1.0))) + ext_bits);
    acc = std::fmin(acc, ext_bits - std::log2((std::pow(m + 0.5, 7.0) / (3.0 * std::pow(rho, 1.5))) * std::pow(lde, 2.0) *
                                              batching_factor(o.batch_d, num_committed)));
    acc = std::fmin(acc, (double)o.grinding - std::log2(std::pow(alpha, q)));
    return sat_u64(acc);
}

// compute_upper_m (security.rs:296-306). Its assert (m_max >= h / 2) holds for every power of two 8 ... 2^32.
static inline double upper_m(uint64_t trace_length) {
    const double h = (double)trace_length;
    const double ratio = (h + 2.0) / h;
    const double m_max = std::ceil(1.0 / (2.0 * (std::sqrt(ratio) - 1.0)));
    return (double)std::min(sat_u64(m_max), MAX_PROXIMITY_PARAMETER);
}

struct Estimate { uint32_t conjectured, ldr, udr; };

// ConjecturedSecurity::compute and ProvenSecurity::compute (security.rs:77-129) with their own arguments. trace_length: a
// power of two >= 8; o: in ProofOptions::new's ranges.
static inline Estimate estimate(const Options& o, uint64_t trace_length, uint32_t collision_res, uint64_t num_constraints,
                                uint64_t num_committed) {
    Estimate e;
    e.conjectured = conjectured(o, collision_res);
    e.udr = (uint32_t)std::min(proven_udr_uncapped(o, trace_length, num_constraints, num_committed), (uint64_t)collision_res);
    const uint32_t m_hi = sat_u32(upper_m(trace_length));
    uint32_t m_opt = 3;
    uint64_t best = 0;
    for (uint32_t m = 3; m < m_hi; m++) {   // max_by_key keeps the last m of the largest value
        const uint64_t v = proven_ldr_at(o, trace_length, m, num_constraints, num_committed);
        if (v >= best) { best = v; m_opt = m; }
    }
    e.ldr = (uint32_t)std::min(proven_ldr_at(o, trace_length, m_opt, num_constraints, num_committed), (uint64_t)collision_res);
    return e;
}

// AcceptableOptions::MinConjecturedSecurity / MinProvenSecurity (verifier/src/lib.rs:333-354): whether the proof passes, and
// the bits the reference's error carries (the conjectured bits, or max(ldr, udr))
static inline bool conjectured_at_least(const Estimate& e, uint32_t bits) { return e.conjectured >= bits; }
static inline bool proven_at_least(const Estimate& e, uint32_t bits) { return e.ldr >= bits || e.udr >= bits; }

// estimates per distinct input within one call: a batch of one AIR pays for one m search per trace length and option set
struct EstimateCache {
    std::map<std::tuple<uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, uint64_t, uint32_t, uint64_t, uint64_t>,
             Estimate> memo;
    Estimate get(const Options& o, uint64_t trace_length, uint32_t collision_res, uint64_t num_constraints, uint64_t num_committed) {
        const auto key = std::make_tuple(o.num_queries, o.blowup, o.grinding, o.ext, o.folding, o.rem_max_deg, o.batch_c, o.batch_d,
                                         trace_length, collision_res, num_constraints, num_committed);
        auto it = memo.find(key);
        if (it == memo.end()) it = memo.emplace(key, estimate(o, trace_length, collision_res, num_constraints, num_committed)).first;
        return it->second;
    }
};

}  // namespace wf_security
