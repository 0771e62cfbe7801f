// tests/fri_ref.cpp — CPU restatement of the standalone FRI prover and verifier: FriProver::build_layers + build_proof with
// DefaultProverChannel, serialized as FriProof, with a tamper hook for dishonest proofs whose every opening verifies, and
// FriVerifier::new + verify with DefaultVerifierChannel; the reference wf_fri_build_proof and wf_fri_verify_batch are tested
// against. TEST INFRASTRUCTURE: compiled by tests/fri_cases.py into a temporary directory, on top of the oracle's field,
// hashes, Merkle trees, folding, coin and tamper list (oracle/wf_prover.cpp, included as one translation unit).
#include "wf_prover.cpp"

// =================================================================================================
// STANDALONE FRI (fri/src/prover/mod.rs:179-296, fri/src/verifier/mod.rs:107-331, fri/src/proof.rs)
// =================================================================================================
namespace {

// FriVerifier verdicts (fri::VerifierError variants the verifier can return), with the layer of InvalidLayerFolding and
// DegreeTruncation in bits 8 and up: the numbering of include/winterfell_b200.h WF_FRI_VERIFY_*
enum { FV_ACCEPT = 0, FV_MALFORMED = 1, FV_LAYER_COMMITMENT = 2, FV_LAYER_FOLDING = 3, FV_REMAINDER_DEGREE = 4,
       FV_REMAINDER_FOLDING = 5, FV_DEGREE_TRUNCATION = 6, FV_RANDOM_COIN = 7 };
static int fv_layer(int code, size_t layer) { return code | (int)(layer << 8); }

// FriProver::build_layers (:179-239) with DefaultProverChannel (coin = new(&[])) kept as state, then build_proof (:254-296)
// serialized as FriProof (proof.rs:149-163,275-285). Tampers: T_FRI_LAYER (layer `index` carries the delta at `row` before
// it is committed, and the next layer is folded from it), T_REMAINDER (delta on coefficient `index`), T_REMAINDER_LONG
// (`index` zero coefficients in front of the remainder). Commitments: the layer roots, then the remainder's.
static std::vector<u8> fri_prove(int h, const u64* evals, size_t len, int d, size_t nf, size_t rem_max_deg, size_t blowup,
                                 const std::vector<u64>& positions, const Tampers* tp, std::vector<u8>& commitments) {
    wfo_coin coin;
    wfo_coin_new(&coin, h, nullptr, 0);
    struct Layer { std::vector<u64> tv; std::vector<u8> leaves, nodes; size_t rows; };
    std::vector<Layer> layers;
    std::vector<u64> cur(evals, evals + len * d);
    size_t cur_len = len;
    const size_t max_rem = (rem_max_deg + 1) * blowup;
    commitments.clear();
    while (cur_len > max_rem) {
        tamper_layer(tp, layers.size(), cur, cur_len, d);
        Layer L;
        L.rows = cur_len / nf;
        L.tv.resize(cur_len * d);
        transpose_slice(cur.data(), cur_len, d, nf, L.tv.data());
        L.leaves.resize(L.rows * 32); L.nodes.resize(L.rows * 32);
        hash_rows(h, L.tv.data(), L.rows, nf * d, nf * d, L.leaves.data());
        merkle_nodes(h, L.leaves.data(), L.rows, L.nodes.data());
        commitments.insert(commitments.end(), L.nodes.data() + 32, L.nodes.data() + 64);
        wfo_coin_reseed(&coin, L.nodes.data() + 32);
        u64 alpha[3] = {0, 0, 0};
        if (coin_draw(&coin, d, alpha)) abort();
        std::vector<u64> nxt(L.rows * d);
        apply_drp(L.tv.data(), L.rows, d, nf, GENERATOR, alpha, nxt.data());
        cur.swap(nxt);
        cur_len = L.rows;
        layers.push_back(std::move(L));
    }
    tamper_layer(tp, layers.size(), cur, cur_len, d);
    auto itw = get_inv_twiddles(cur_len);
    interpolate_poly_with_offset(cur.data(), cur_len, d, itw.data(), GENERATOR);
    const size_t rs = cur_len / blowup;
    std::vector<u64> remainder(rs * d);
    for (size_t i = 0; i < rs; i++) for (int k = 0; k < d; k++) remainder[i * d + k] = cur[(rs - 1 - i) * d + k];
    if (tp)
        for (const Tamper& t : tp->list) {
            if (t.target == T_REMAINDER)
                for (int k = 0; k < d; k++) remainder[t.index * d + k] = f_add(remainder[t.index * d + k], t.delta[k]);
            if (t.target == T_REMAINDER_LONG) remainder.insert(remainder.begin(), t.index * d, 0);
        }
    u8 dg[32];
    hash_elements(h, remainder.data(), remainder.size(), dg);
    commitments.insert(commitments.end(), dg, dg + 32);
    Writer w;
    w.u8_((u8)layers.size());
    std::vector<u64> p = positions;
    size_t dom = len;
    for (auto& L : layers) {
        std::vector<u64> fp(p.size());
        fp.resize(fold_positions(p.data(), p.size(), dom, nf, fp.data()));
        p = fp;
        Writer vals;
        for (u64 q : p) vals.bytes(&L.tv[q * nf * d], nf * d * 8);
        std::vector<u8> lv(p.size() * 32), pr(64 + p.size() * 40 * 33);
        long pl = merkle_prove_batch(L.leaves.data(), L.nodes.data(), L.rows, p.data(), p.size(), lv.data(), pr.data(), pr.size(),
                                     digest_len(h));
        if (pl < 0) abort();
        w.u32_((u32)vals.b.size()); w.bytes(vals.b.data(), vals.b.size());
        w.u32_((u32)pl); w.bytes(pr.data(), (size_t)pl);
        dom /= nf;
    }
    w.u16_((uint16_t)(remainder.size() * 8)); w.bytes(remainder.data(), remainder.size() * 8);
    w.u8_(0);   // log2(num_partitions = 1)
    return w.b;
}

// DefaultVerifierChannel::new (verifier/channel.rs:146-170) + FriVerifier::new (:107-152) + verify (:199-331). Returns a
// verdict (FV_*). The caller checked the shape, the positions (< domain) and the evaluations (canonical), and that there
// are num_layers + 1 commitments.
static int fri_verify(int h, int d, size_t nf, size_t max_deg, size_t domain, size_t nl, const u8* proof, size_t len,
                      const u8* cms, const u8* seed, const u64* positions, const u64* evaluations, size_t k) {
    Field F{d};
    // FriProof::read_from (proof.rs:166-179), then parse_remainder and parse_layers (proof.rs:98-146); read_from_bytes
    // refuses bytes after the proof
    Reader r{proof, len};
    const u8 nlay = r.u8_();
    std::vector<std::vector<u8>> fv, fp;
    for (u32 i = 0; i < nlay && r.ok; i++) {
        const u64 vn = r.le(4);
        const u8* v = r.take(vn);
        if (!r.ok || vn == 0) return FV_MALFORMED;
        const u64 pn = r.le(4);
        const u8* pp = r.take(pn);
        if (!r.ok) return FV_MALFORMED;
        fv.emplace_back(v, v + vn);
        fp.emplace_back(pp, pp + pn);
    }
    const u64 rl = r.le(2);
    const u8* rem = r.take(rl);
    const u8 log_parts = r.u8_();
    if (!r.ok || r.pos != len) return FV_MALFORMED;
    if (log_parts >= 64) return FV_MALFORMED;   // 2usize.pow(num_partitions) does not fit a usize
    const size_t rn = rl / (8 * d);
    if (rn == 0 || (rn & (rn - 1)) || rl % (8 * d) || !words_canonical(rem, rl)) return FV_MALFORMED;
    std::vector<BatchProof> bps(nlay);
    {
        size_t ds = domain;
        for (size_t i = 0; i < nlay; i++) {
            ds /= nf;
            if (fv[i].size() % (8 * d * nf) || !words_canonical(fv[i].data(), fv[i].size())) return FV_MALFORMED;
            Reader pr{fp[i].data(), fp[i].size()};
            if (!read_batch_proof(pr, bps[i], h) || pr.pos != fp[i].size() || ((size_t)1 << bps[i].depth) != ds) return FV_MALFORMED;
        }
    }
    // FriVerifier::new: reseed with every commitment and draw its alpha
    wfo_coin coin;
    if (seed) { memcpy(coin.seed, seed, 32); coin.counter = 0; coin.hash_id = h; }
    else wfo_coin_new(&coin, h, nullptr, 0);
    std::vector<std::array<u8, 32>> cm(nl + 1);
    for (size_t i = 0; i <= nl; i++) {
        cm[i].fill(0);
        memcpy(cm[i].data(), cms + 32 * i, digest_len(h));
        reduce_digest(h, cm[i].data());
    }
    std::vector<EE> alphas;
    size_t mdp1 = max_deg + 1;
    for (size_t i = 0; i <= nl; i++) {
        wfo_coin_reseed(&coin, cm[i].data());
        EE a = F.zero();
        if (coin_draw(&coin, d, a.v)) return FV_RANDOM_COIN;
        alphas.push_back(a);
        if (i != nl && mdp1 % nf) return fv_layer(FV_DEGREE_TRUNCATION, i);
        mdp1 /= nf;
    }
    // verify_generic
    std::vector<u64> pos(positions, positions + k);
    std::vector<EE> evals(k);
    for (size_t i = 0; i < k; i++) { evals[i] = F.zero(); memcpy(evals[i].v, evaluations + i * d, 8 * d); }
    const u64 P_ = (u64)1 << log_parts;
    size_t dom = domain;
    u64 dg = root_of_unity((u32)__builtin_ctzll(domain));
    mdp1 = max_deg + 1;
    for (size_t depth = 0; depth < nl; depth++) {
        const size_t row_len = dom / nf;
        std::vector<u64> fpos(pos.size());
        fpos.resize(fold_positions(pos.data(), pos.size(), dom, nf, fpos.data()));
        // map_positions_to_indexes (fri/src/utils.rs:9-33)
        std::vector<u64> idx = fpos;
        if (P_ > 1) {
            const u64 psize = row_len / P_;
            for (auto& q : idx) q = (q % P_) * psize + (q - q % P_) / P_;
            std::set<u64> seen(idx.begin(), idx.end());
            if (seen.size() != idx.size() || (!seen.empty() && *seen.rbegin() >= row_len)) return FV_MALFORMED;   // leaves the tree
        }
        if (depth >= nlay) return FV_MALFORMED;   // the proof has no layer left to read
        const std::vector<u8>& vals = fv[depth];
        const size_t rows = vals.size() / (8 * d * nf);
        std::vector<std::array<u8, 32>> lv(rows);
        for (size_t i = 0; i < rows; i++) hash_elements(h, (const u64*)(vals.data() + i * nf * d * 8), nf * d, lv[i].data());
        u8 got[32];
        if (!batch_root(h, bps[depth], idx, lv, got) || memcmp(got, cm[depth].data(), 32)) return FV_LAYER_COMMITMENT;
        for (size_t i = 0; i < pos.size(); i++) {   // get_query_values (:335-351)
            const size_t at = std::find(fpos.begin(), fpos.end(), pos[i] % row_len) - fpos.begin();
            EE v = F.zero();
            memcpy(v.v, vals.data() + (at * nf + pos[i] / row_len) * d * 8, d * 8);
            if (!F.eq(v, evals[i])) return fv_layer(FV_LAYER_FOLDING, depth);
        }
        // each queried row interpolated over {x_e w_nf^r} and evaluated at alpha: apply_drp on one row (folding/mod.rs:86-118)
        std::vector<EE> nxt(fpos.size());
        const auto itw = get_inv_twiddles(nf);
        for (size_t i = 0; i < fpos.size(); i++) {
            std::vector<u64> row(nf * d);
            memcpy(row.data(), vals.data() + i * nf * d * 8, nf * d * 8);
            const u64 xinv = f_inv(f_mul(f_exp(dg, fpos[i]), GENERATOR));
            ref_fft_in_place(row.data(), nf, d, itw.data());
            permute_words(row.data(), nf, d);
            u64 off = f_inv((u64)nf);
            std::vector<EE> coefs(nf);
            for (size_t j = 0; j < nf; j++) {
                coefs[j] = F.zero();
                for (int q = 0; q < d; q++) coefs[j].v[q] = f_mul(row[j * d + q], off);
                off = f_mul(off, xinv);
            }
            nxt[i] = horner_ext(F, coefs.data(), nf, alphas[depth]);
        }
        if (mdp1 % nf) return fv_layer(FV_DEGREE_TRUNCATION, depth);   // new() refused these already
        evals = nxt;
        pos = fpos;
        dg = f_exp(dg, nf);
        mdp1 /= nf;
        dom = row_len;
    }
    if (rn > mdp1) return FV_REMAINDER_DEGREE;
    for (size_t i = 0; i < pos.size(); i++) {   // eval_horner_rev at offset * g^position
        const u64 x = f_mul(f_exp(dg, pos[i]), GENERATOR);
        EE acc = F.zero();
        for (size_t j = 0; j < rn; j++) {
            EE cj = F.zero();
            memcpy(cj.v, rem + j * d * 8, d * 8);
            acc = F.add(F.mul_base(acc, x), cj);
        }
        if (!F.eq(acc, evals[i])) return FV_REMAINDER_FOLDING;
    }
    return FV_ACCEPT;
}

// the shape of FriVerifier::new: the domain max_deg.next_power_of_two() * blowup and its number of layers; false when
// the options cannot describe a FRI proof (every layer needs a tree of two leaves or more, and a remainder of one element
// or more)
static bool fri_shape(size_t nf, size_t rem_max_deg, size_t blowup, size_t max_deg, size_t* domain, size_t* nl) {
    if (blowup == 0 || (blowup & (blowup - 1)) || max_deg >= ((size_t)1 << 32)) return false;
    size_t np2 = 1;
    while (np2 < max_deg) np2 <<= 1;   // usize::next_power_of_two (0 -> 1)
    if (np2 * blowup > ((size_t)1 << 32)) return false;
    size_t dom = np2 * blowup, n = 0;
    const size_t max_rem = (rem_max_deg + 1) * blowup;
    while (dom > max_rem) {
        if (dom / nf < 2) return false;
        dom /= nf;
        n++;
    }
    if (dom / blowup == 0) return false;
    *domain = np2 * blowup;
    *nl = n;
    return true;
}

}  // namespace

extern "C" {
// Standalone FRI prover: the commit phase of the oracle's wfo_fri_build_layers (same arguments), then FriProver::build_proof
// at `positions` (k words, any order, repeats allowed). commitments_out: (num_layers + 1) x 32 bytes. tamper: [ntamper][6] words as for the
// proving entry points, targets T_FRI_LAYER, T_REMAINDER, T_REMAINDER_LONG. Returns the proof length, -1 when it does not fit
// `cap`, -4 for a tamper that does not fit the proof.
long wfr_fri_build_proof(int hash_id, const uint64_t* evals, size_t len, int d, size_t folding, size_t rem_max_deg, size_t blowup,
                         const uint64_t* positions, size_t k, const uint64_t* tamper, size_t ntamper, uint8_t* commitments_out,
                         uint8_t* out, size_t cap) {
    Tampers tp;
    const size_t nl = fri_num_layers(len, folding, rem_max_deg, blowup);
    size_t last = len;
    for (size_t i = 0; i < nl; i++) last /= folding;
    for (size_t i = 0; i < ntamper; i++) {
        const uint64_t* t = tamper + 6 * i;
        Tamper x{t[0], t[1], t[2], {t[3], t[4], t[5]}};
        size_t ll = len;
        for (u64 q = 0; q < x.index && q < nl; q++) ll /= folding;
        const bool all = x.row == ALL_ROWS;
        if (x.delta[0] >= P || x.delta[1] >= P || x.delta[2] >= P) return -4;
        if (x.target == T_FRI_LAYER && (x.index > nl || (!all && x.row >= ll))) return -4;
        if (x.target == T_REMAINDER && (x.index >= last / blowup || !all)) return -4;
        if (x.target == T_REMAINDER_LONG && (x.index < 1 || x.index > 4096 || !all)) return -4;
        if (x.target != T_FRI_LAYER && x.target != T_REMAINDER && x.target != T_REMAINDER_LONG) return -4;
        tp.list.push_back(x);
    }
    std::vector<u8> cm;
    std::vector<u8> p = fri_prove(hash_id, evals, len, d, folding, rem_max_deg, blowup, std::vector<u64>(positions, positions + k),
                                  ntamper ? &tp : nullptr, cm);
    if (p.size() > cap) return -1;
    memcpy(out, p.data(), p.size());
    memcpy(commitments_out, cm.data(), cm.size());
    return (long)p.size();
}
// FriVerifier::new + verify with DefaultVerifierChannel for one FriProof: commitments = num_commitments x 32 bytes (layer roots,
// then the remainder's), coin_seed = the public coin's 32-byte seed (NULL: DefaultRandomCoin::new(&[])), positions and
// evaluations ([k][d] canonical words). Returns the verdict (WF_FRI_VERIFY_* of include/winterfell_b200.h), -1 for arguments
// that describe no proof (a shape with no layer tree or remainder, a commitment count other than num_layers + 1, a position
// outside the domain, a non-canonical evaluation), -2 for a folding factor other than 2, 4, 8 or 16.
int wfr_fri_verify(int hash_id, int d, size_t folding, size_t rem_max_deg, size_t blowup, size_t max_poly_degree, const uint8_t* proof,
                   size_t len, const uint8_t* commitments, size_t num_commitments, const uint8_t* coin_seed, const uint64_t* positions,
                   const uint64_t* evaluations, size_t k) {
    if (folding != 2 && folding != 4 && folding != 8 && folding != 16) return -2;
    size_t domain, nl;
    if (d < 1 || d > 3 || !fri_shape(folding, rem_max_deg, blowup, max_poly_degree, &domain, &nl) || num_commitments != nl + 1)
        return -1;
    for (size_t i = 0; i < k; i++) {
        if (positions[i] >= domain) return -1;
        for (int q = 0; q < d; q++) if (evaluations[i * d + q] >= P) return -1;
    }
    return fri_verify(hash_id, d, folding, max_poly_degree, domain, nl, proof, len, commitments, coin_seed, positions, evaluations, k);
}
}
