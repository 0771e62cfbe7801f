// host_transcript.hpp — host-side hashing, random coin and byte writer of the product.
//
// The Fiat-Shamir transcript is tiny, strictly sequential and must be bit-exact, so it stays on
// the host (SURVEY.md §1 "sideways, not accelerated"). Follows crypto/src/hash/mod.rs:31-64
// (Hasher / ElementHasher), crypto/src/random/default.rs:82-247 (DefaultRandomCoin) and
// utils/core/src/serde/byte_writer.rs:77-92,145-149 (vint64 usize encoding).
#pragma once
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "blake3.cuh"
#include "commit.cuh"
#include "rp64.cuh"
#include "rpjive.cuh"
#include "sha3.cuh"

struct Digest {
    u8 b[32];
};

// (digests live in 32-byte slots; Blake3_192 keeps the first 24 bytes, the rest of the slot is zero — commit.cuh)
static inline Digest hh_hash_elements(int hash_id, const u64* e, size_t n) {
    Digest d;
    if (WF_HASH_IS_BLAKE3(hash_id)) {
        b3_host_hash(reinterpret_cast<const u8*>(e), n * 8, d.b);  // canonical LE bytes (x86 host is LE)
        if (hash_id == WF_HASH_BLAKE3_192) memset(d.b + 24, 0, 8);
    } else {
        u64 o[4];
        if (hash_id == WF_HASH_RP64_256) rp64_host_hash_elements(e, n, o);
        else if (hash_id == WF_HASH_SHA3_256) sha3_host_words(e, n, o);   // sha/mod.rs:49-55: the canonical LE element bytes
        else rpj_host_hash_elements(e, n, o);
        memcpy(d.b, o, 32);
    }
    return d;
}
static inline Digest hh_merge(int hash_id, const Digest& a, const Digest& b) {
    Digest d;
    if (WF_HASH_IS_BLAKE3(hash_id)) {
        const size_t dl = WF_DIGEST_BYTES(hash_id);   // blake/mod.rs:33, :85-88: the digests' bytes back to back
        u8 two[64];
        memcpy(two, a.b, dl);
        memcpy(two + dl, b.b, dl);
        b3_host_hash(two, 2 * dl, d.b);
        if (dl == 24) memset(d.b + 24, 0, 8);
    } else {
        u64 in[8], o[4];
        memcpy(in, a.b, 32);
        memcpy(in + 4, b.b, 32);
        if (hash_id == WF_HASH_RP64_256) rp64_merge(in, o);
        else if (hash_id == WF_HASH_SHA3_256) sha3_host_words(in, 8, o);
        else rpj_merge(in, o);
        memcpy(d.b, o, 32);
    }
    return d;
}
static inline Digest hh_merge_with_int(int hash_id, const Digest& seed, u64 value) {
    Digest d;
    if (WF_HASH_IS_BLAKE3(hash_id)) {
        const size_t dl = WF_DIGEST_BYTES(hash_id);   // blake/mod.rs:41-46, :95-102
        u8 data[40];
        memcpy(data, seed.b, dl);
        memcpy(data + dl, &value, 8);
        b3_host_hash(data, dl + 8, d.b);
        if (dl == 24) memset(d.b + 24, 0, 8);
    } else {
        u64 s[4], o[4];
        memcpy(s, seed.b, 32);
        if (hash_id == WF_HASH_RP64_256) rp64_host_merge_with_int(s, value, o);
        else if (hash_id == WF_HASH_SHA3_256) { u64 w5[5] = {s[0], s[1], s[2], s[3], value}; sha3_host_words(w5, 5, o); }
        else rpj_merge_with_int(s, value, o);
        memcpy(d.b, o, 32);
    }
    return d;
}

// DefaultRandomCoin (crypto/src/random/default.rs)
struct PublicCoin {
    int hash_id;
    Digest seed;
    u64 counter;
    PublicCoin(int h, const u64* seed_elems, size_t n) : hash_id(h), counter(0) { seed = hh_hash_elements(h, seed_elems, n); }
    void reseed(const Digest& data) {  // :131-134
        seed = hh_merge(hash_id, seed, data);
        counter = 0;
    }
    void reseed_with_int(u64 v) {  // draw_integers prologue :223-225
        seed = hh_merge_with_int(hash_id, seed, v);
        counter = 0;
    }
    Digest next() {  // :82-85
        counter += 1;
        return hh_merge_with_int(hash_id, seed, counter);
    }
    // draw an element of extension degree d (:156-170); any word >= p rejects the whole draw
    bool draw(int d, u64* out) {
        for (int t = 0; t < 1000; t++) {
            Digest v = next();
            u64 w[3];
            memcpy(w, v.b, 8 * d);
            bool ok = true;
            for (int k = 0; k < d; k++) ok = ok && w[k] < GL_P;
            if (ok) {
                for (int k = 0; k < d; k++) out[k] = w[k];
                return true;
            }
        }
        return false;
    }
    u32 check_leading_zeros(u64 value) const {  // :141-146
        Digest s = hh_merge_with_int(hash_id, seed, value);
        u64 head;
        memcpy(&head, s.b, 8);
        return head == 0 ? 64 : (u32)__builtin_ctzll(head);
    }
    bool draw_integers(size_t num, size_t domain, u64 nonce, std::vector<u64>& out) {  // :210-247
        reseed_with_int(nonce);
        u64 mask = (u64)domain - 1;
        out.clear();
        for (int t = 0; t < 1000 && out.size() < num; t++) {
            Digest v = next();
            u64 x;
            memcpy(&x, v.b, 8);
            out.push_back(x & mask);
        }
        return out.size() == num;
    }
};

// the query positions over a domain of `domain` points (prover/src/channel.rs:150-163, verifier/src/lib.rs:284-292):
// draw_integers, then sorted and deduplicated. false when the coin cannot draw them.
static inline bool query_positions(PublicCoin& coin, size_t num_queries, size_t domain, u64 nonce, std::vector<u64>& pos) {
    if (!coin.draw_integers(num_queries, domain, nonce, pos)) return false;
    std::sort(pos.begin(), pos.end());
    pos.erase(std::unique(pos.begin(), pos.end()), pos.end());
    return true;
}
// fold_positions (fri/src/folding/mod.rs:159-176): the positions' rows in a layer of row_len rows, first occurrences in order
static inline std::vector<u64> fold_positions(const std::vector<u64>& pos, size_t row_len) {
    std::vector<u64> r;
    for (u64 p : pos)
        if (std::find(r.begin(), r.end(), p % row_len) == r.end()) r.push_back(p % row_len);
    return r;
}

// ByteWriter (utils/core/src/serde/byte_writer.rs)
struct ByteVec {
    std::vector<u8> v;
    void u8_(u8 x) { v.push_back(x); }
    void u16_(uint16_t x) { for (int i = 0; i < 2; i++) v.push_back((u8)(x >> (8 * i))); }
    void u32_(u32 x) { for (int i = 0; i < 4; i++) v.push_back((u8)(x >> (8 * i))); }
    void u64_(u64 x) { for (int i = 0; i < 8; i++) v.push_back((u8)(x >> (8 * i))); }
    void bytes(const void* p, size_t n) { const u8* q = (const u8*)p; v.insert(v.end(), q, q + n); }
    void usize(u64 value) {  // vint64, :77-92 and usize_encoded_len :145-149
        int zeros = value == 0 ? 64 : __builtin_clzll(value);
        int len = 9 - ((zeros > 0 ? zeros - 1 : 0) / 7 < 8 ? (zeros > 0 ? zeros - 1 : 0) / 7 : 8);
        if (len == 9) {
            u8_(0);
            u64_(value);
        } else {
            u64 enc = ((value << 1) | 1) << (len - 1);
            for (int i = 0; i < len; i++) v.push_back((u8)(enc >> (8 * i)));
        }
    }
};
