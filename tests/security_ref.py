"""An independent Python restatement of the reference's security estimator (air/src/proof/security.rs:20-306):
ConjecturedSecurity::compute, ProvenSecurity::compute and the acceptance rules of AcceptableOptions (verifier/src/lib.rs:
333-358), for the Goldilocks field. The libm calls and their order are the reference's: math.log2 / math.pow / math.sqrt /
math.ceil call the same C library functions as Rust's f64::log2 / powf / sqrt / ceil. Where Python raises and Rust returns an
IEEE value (log2 of 0 or of a negative number), this module returns what Rust returns, and float-to-integer casts saturate as
Rust's `as` does (NaN -> 0)."""
import math

BASE_FIELD_BITS = 64                 # Goldilocks: Context::num_modulus_bits of 2^64 - 2^32 + 1
GRINDING_CONTRIBUTION_FLOOR = 80
MAX_PROXIMITY_PARAMETER = 1000
U64_MAX = (1 << 64) - 1
U32_MAX = (1 << 32) - 1

# Hasher::COLLISION_RESISTANCE by winterfell_b200 hash id (crypto/src/hash/blake/mod.rs:27,79; rp64_256/mod.rs:121;
# rp64_256_jive/mod.rs:117; sha/mod.rs:24)
COLLISION_RESISTANCE = {0: 128, 1: 128, 2: 128, 3: 96, 4: 128}

LINEAR, ALGEBRAIC, HORNER = 0, 1, 2


def log2(x):
    """f64::log2: -inf at 0, NaN below 0 and for NaN."""
    if math.isnan(x) or x < 0:
        return math.nan
    if x == 0:
        return -math.inf
    return math.log2(x)


def fmin(a, b):
    """f64::min: the other operand when one is NaN."""
    if math.isnan(a):
        return b
    if math.isnan(b):
        return a
    return a if a < b else b


def sat(x, hi):
    """`x as u64` / `x as u32`: NaN and negatives to 0, values above the range to its maximum, truncation toward zero."""
    if math.isnan(x) or x <= 0:
        return 0
    if x >= hi + 1:
        return hi
    return int(x)


def fold_min(eps):
    acc = math.inf
    for e in eps:
        acc = fmin(acc, e)
    return acc


def num_fri_layers(domain, folding, rem_max_deg, blowup):
    """FriOptions::num_fri_layers (fri/src/options.rs:85-93)."""
    n, mx = 0, (rem_max_deg + 1) * blowup
    while domain > mx:
        domain //= folding
        n += 1
    return n


def conjectured(ext, blowup, num_queries, grinding, collision_resistance):
    """ConjecturedSecurity::compute (security.rs:30-47)."""
    field_security = BASE_FIELD_BITS * ext
    query_security = (blowup.bit_length() - 1) * num_queries
    if query_security >= GRINDING_CONTRIBUTION_FLOOR:
        query_security += grinding
    return min(min(field_security, query_security) - 1, collision_resistance)


def batching_factor(method, count):
    return 1.0 if method == LINEAR else float(count) - 1.0


def proven_udr(o, trace_length, num_constraints, num_committed_polys):
    """proven_security_protocol_unique_decoding (security.rs:223-285), before the cap."""
    ext_bits = float(BASE_FIELD_BITS * o["ext"])
    q = float(o["num_queries"])
    lde = float(trace_length * o["blowup"])
    h = float(trace_length)
    num_openings = 2.0
    rho_plus = (h + num_openings) / lde
    alpha = (1.0 + rho_plus) * 0.5
    max_deg = float(o["blowup"]) + 1.0
    eps = []
    eps.append(-log2(batching_factor(o["batch_c"], num_constraints)) + ext_bits)
    eps.append(-log2(max_deg * (h + num_openings - 1.0) + (h - 1.0)) + ext_bits)
    eps.append(ext_bits - log2(lde * batching_factor(o["batch_d"], num_committed_polys)))
    folding = float(o["folding"])
    nl = num_fri_layers(trace_length * o["blowup"], o["folding"], o["rem_max_deg"], o["blowup"])
    eps.append(fold_min(ext_bits - log2((folding - 1.0) * (lde + 1.0)) for _ in range(nl)))
    eps.append(float(o["grinding"]) - log2(math.pow(alpha, q)))
    return sat(fold_min(eps), U64_MAX)


def proven_ldr_at(o, trace_length, m, num_constraints, num_committed_polys):
    """proven_security_protocol_for_given_proximity_parameter (security.rs:150-220)."""
    ext_bits = float(BASE_FIELD_BITS * o["ext"])
    q = float(o["num_queries"])
    m = float(m)
    rho = 1.0 / float(o["blowup"])
    alpha = (1.0 + 0.5 / m) * math.sqrt(rho)
    max_deg = float(o["blowup"]) + 1.0
    lde = float(trace_length * o["blowup"])
    h = float(trace_length)
    num_openings = 2.0
    den = rho - (2.0 * m / lde)
    if den == 0.0:           # m / 0 in IEEE arithmetic (m > 0)
        l = math.inf if math.copysign(1.0, den) > 0 else -math.inf
    else:
        l = m / den
    eps = []
    eps.append(-log2(l) - log2(batching_factor(o["batch_c"], num_constraints)) + ext_bits)
    eps.append(-log2(l * l * (max_deg * (h + num_openings - 1.0) + (h - 1.0))) + ext_bits)
    eps.append(ext_bits - log2((math.pow(m + 0.5, 7.0) / (3.0 * math.pow(rho, 1.5))) * math.pow(lde, 2.0)
                               * batching_factor(o["batch_d"], num_committed_polys)))
    eps.append(float(o["grinding"]) - log2(math.pow(alpha, q)))
    return sat(fold_min(eps), U64_MAX)


def upper_m(h):
    """compute_upper_m (security.rs:296-306); None where the reference's assert fails."""
    h = float(h)
    ratio = (h + 2.0) / h
    m_max = math.ceil(1.0 / (2.0 * (math.sqrt(ratio) - 1.0)))
    if not m_max >= h / 2.0:
        return None
    return float(min(sat(float(m_max), U64_MAX), MAX_PROXIMITY_PARAMETER))


def proven(o, trace_length, collision_resistance, num_constraints, num_committed_polys):
    """ProvenSecurity::compute (security.rs:77-129): (udr, ldr)."""
    udr = min(proven_udr(o, trace_length, num_constraints, num_committed_polys), collision_resistance)
    m_max = upper_m(trace_length)
    assert m_max is not None, trace_length
    best, best_key = None, -1
    for m in range(3, sat(m_max, U32_MAX)):          # max_by_key: the last m with the largest value
        k = proven_ldr_at(o, trace_length, m, num_constraints, num_committed_polys)
        if k >= best_key:
            best, best_key = m, k
    assert best is not None
    ldr = min(proven_ldr_at(o, trace_length, best, num_constraints, num_committed_polys), collision_resistance)
    return udr, ldr


def opts_dict(words):
    """The option fields the estimate reads from the opts[9] words of the C ABI."""
    keys = ("num_queries", "blowup", "grinding", "ext", "folding", "rem_max_deg", "batch_c", "batch_d")
    return dict(zip(keys, (int(w) for w in words[:8])))


def estimate(words, trace_length, collision_resistance, num_constraints, num_committed_polys):
    """(conjectured, proven ldr, proven udr), the outputs of wf_security_estimate."""
    o = opts_dict(words)
    c = conjectured(o["ext"], o["blowup"], o["num_queries"], o["grinding"], collision_resistance)
    udr, ldr = proven(o, trace_length, collision_resistance, num_constraints, num_committed_polys)
    return c, ldr, udr
