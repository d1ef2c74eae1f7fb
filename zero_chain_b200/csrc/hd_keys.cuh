// Wallet keys: zface's hierarchical key derivation (a ZIP-32-style scheme, zface/src/derive/mod.rs) with the Diversifier
// generator P_G.  Restates, value for value:
//   prf_expand_vec(k, ts)        BLAKE2b-512 "zech_ExpandSeed_" (k || ts...)               core/proofs/src/no_std_aliases/keys.rs:25-40
//   ExtendedSpendingKey::master  I = BLAKE2b-512 "Zerochain_Master" (seed); sk = SpendingKey::from_seed(I_L), chain code
//                                I_R, depth 0, parent tag 0, child index 0                derive/mod.rs:48-64
//   ExtendedSpendingKey::derive_child(i), pgk = sk P_G of the parent
//                                hardened (i >= 2^31): I = prf_expand_vec(c, [0x11, sk, i LE])
//                                otherwise:            I = prf_expand_vec(c, [0x12, Point::write(pgk), i LE])
//                                child sk = to_uniform(prf_expand(I_L, [0x13])) + sk, chain code I_R, depth + 1, index i,
//                                parent tag = the first 4 bytes of BLAKE2b-256 "ZerochainEFinger" (Point::write(pgk))
//                                derive/mod.rs:66-104, components.rs:15-35
//   ExtendedProofGenerationKey::derive_child(i)
//                                hardened i is an error; child pgk = to_uniform(prf_expand(I_L, [0x13])) P_G + pgk, with I,
//                                tag, depth and chain code as above                        derive/mod.rs:164-197
//   From<&ExtendedSpendingKey>   the same header with key = sk P_G                         derive/mod.rs:136-146
//   write / read                 depth u8 | parent tag 4 B | child index u32 LE | chain code 32 B | key 32 B (73 B), the key
//                                an sk (SpendingKey::read: < r_J) or a pgk (ProofGenerationKey::read: Point::read +
//                                as_prime_order)                                           derive/mod.rs:106-133, 199-227
// and an account's dk = into_decryption_key(pgk) and ek = dk P_G (decryption_key / pg_mul of tx_build.cuh).
//
// Every message is at most 69 bytes, so each hash is one BLAKE2b compression built straight from registers.  A depth of
// 255 is refused: the reference's depth + 1 on a u8 panics in a debug build and wraps in a release build.
//
// Everything is inlined into the kernels (hd_keys.cu), with the same rules as tx_build.cuh: thread-local arrays are
// indexed only with compile-time constants, so nothing goes to local memory.  The same source compiles with ZK_HOST_EMUL for
// the CPU test (tests/host_emul/emul_hd_keys.cpp).
#pragma once
#include "tx_build.cuh"

namespace zkhd {
using namespace zktb;

constexpr int HD_XK_BYTES = 73;                              // one extended key, written
constexpr int HD_TAG = 1, HD_INDEX = 5, HD_CHAIN = 9, HD_KEY = 41;   // byte offsets of its fields
constexpr int HD_BAD_INDEX = 4, HD_HARDENED = 5, HD_DEPTH = 6;       // row statuses besides the zk_jubjub_into_xy codes
constexpr uint32_t HD_HARDENED_BIT = 0x80000000u;
constexpr uint32_t HD_MAX_DEPTH = 254;                       // the deepest parent a child can be derived from
// "Zerochain_Master" and "ZerochainEFinger" (zface/src/derive/constants.rs) as two little-endian words each
constexpr uint64_t HD_MASTER0 = 0x696168636f72655aull, HD_MASTER1 = 0x72657473614d5f6eull;
constexpr uint64_t HD_FINGER0 = 0x696168636f72655aull, HD_FINGER1 = 0x7265676e6946456eull;

// ---- hashes ---------------------------------------------------------------------------------------------------------------
// BLAKE2b with an empty key and salt, a 16-byte personalization and a dlen-byte digest of a message of len <= 128 bytes
// held in m (zero past the end); the digest is the first dlen / 8 words of h
ZK_DEV void b2b_single(uint64_t pers0, uint64_t pers1, uint32_t dlen, const uint64_t *m, uint64_t len, uint64_t *h) {
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = b2b_iv(i);
    h[0] ^= 0x01010000ull | dlen;                 // digest length, key length 0, fanout 1, depth 1
    h[6] ^= pers0;
    h[7] ^= pers1;
    b2b_compress(h, m, len, true);
}
ZK_DEV uint64_t hd_word(const uint32_t *w, int i) { return (uint64_t)w[2 * i] | ((uint64_t)w[2 * i + 1] << 32); }

// EncKeyFingerPrint::tag: the first 4 bytes of BLAKE2b-256 "ZerochainEFinger" of a pgk encoding, as a little-endian word
ZK_DEV uint32_t hd_tag(const uint32_t *pgk) {
    uint64_t m[16], h[8];
#pragma unroll
    for (int w = 0; w < 16; w++) m[w] = w < 4 ? hd_word(pgk, w & 3) : 0;
    b2b_single(HD_FINGER0, HD_FINGER1, 32, m, 32, h);
    return (uint32_t)h[0];
}

// prf_expand_vec(c, [t, key, index LE]): BLAKE2b-512 of the 69 bytes c || t || key || index (c and key 8 words each)
ZK_DEV void hd_prf_child(const uint32_t *c, uint32_t t, const uint32_t *key, uint32_t index, uint64_t *h) {
    uint32_t s[10];                               // t || key || index: 37 bytes as 10 little-endian words
    s[0] = t | (key[0] << 8);
#pragma unroll
    for (int i = 1; i < 8; i++) s[i] = (key[i - 1] >> 24) | (key[i] << 8);
    s[8] = (key[7] >> 24) | (index << 8);
    s[9] = index >> 24;
    uint64_t m[16];
#pragma unroll
    for (int w = 0; w < 16; w++) m[w] = w < 4 ? hd_word(c, w & 3) : w < 9 ? hd_word(s, (w + 1) % 5) : 0;
    b2b_single(TB_EXPAND0, TB_EXPAND1, 64, m, 69, h);
}

// to_uniform(prf_expand(I_L, [0x13])): the scalar a child adds to its parent's key (I: the 8 digest words of hd_prf_child)
ZK_DEV Fs hd_tweak(const uint64_t *I) {
    uint64_t m[16], h[8];
#pragma unroll
    for (int w = 0; w < 16; w++) m[w] = w < 4 ? I[w & 3] : w == 4 ? 0x13 : 0;
    b2b_single(TB_EXPAND0, TB_EXPAND1, 64, m, 33, h);
    return fs_to_uniform(h);
}

// ExtendedSpendingKey::master(seed): the master sk, and the chain code I_R in chain (8 words)
ZK_DEV Fs hd_master(const uint8_t *seed, uint64_t len, uint32_t *chain) {
    uint64_t I[8], m[16], h[8];
    b2b_prefixed<0>(HD_MASTER0, HD_MASTER1, nullptr, seed, len, I);
#pragma unroll
    for (int i = 0; i < 4; i++) { chain[2 * i] = (uint32_t)I[4 + i]; chain[2 * i + 1] = (uint32_t)(I[4 + i] >> 32); }
#pragma unroll
    for (int w = 0; w < 16; w++) m[w] = w < 4 ? I[w & 3] : 0;
    b2b_single(TB_EXPAND0, TB_EXPAND1, 64, m, 32, h);   // SpendingKey::from_seed(I_L)
    return fs_to_uniform(h);
}

// ---- the 73-byte layout -----------------------------------------------------------------------------------------------------
ZK_DEV void hd_load(const uint8_t *b, uint32_t *w) {   // 8 little-endian words from bytes (any alignment)
#pragma unroll
    for (int i = 0; i < 8; i++)
        w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
}
ZK_DEV void hd_put_u32(uint8_t *b, uint32_t v) {
#pragma unroll
    for (int k = 0; k < 4; k++) b[k] = (uint8_t)(v >> (8 * k));
}
ZK_DEV void hd_zero(uint8_t *b, int n) {
    if (b)
        for (int i = 0; i < n; i++) b[i] = 0;
}
// an extended key: depth | parent tag | child index | chain code | key
ZK_DEV void hd_put(uint8_t *out, uint32_t depth, uint32_t tag, uint32_t index, const uint32_t *chain, const uint32_t *key) {
    out[0] = (uint8_t)depth;
    hd_put_u32(out + HD_TAG, tag);
    hd_put_u32(out + HD_INDEX, index);
    store_le_words(out + HD_CHAIN, chain, 8);
    store_le_words(out + HD_KEY, key, 8);
}

// ---- an account's keys ------------------------------------------------------------------------------------------------------
// dk = into_decryption_key and ek = dk P_G of the account whose pgk encodes to pgk; each output may be NULL
ZK_DEV void hd_dk_ek(const uint32_t *pgk, uint8_t *dk_out, uint8_t *ek_out) {
    uint32_t h[8];
    b2s_256(TB_BDK0, TB_BDK1, 32, [&](uint32_t k) { return k < 8 ? pgk[k & 7] : 0u; }, h);
    h[7] &= 0x07ffffffu;
    if (dk_out) store_le_words(dk_out, h, 8);
    if (ek_out) {
        uint32_t e[8];
        ext_encode(pg_mul(fs_words(h)), e);
        store_le_words(ek_out, e, 8);
    }
}
// An extended spending key and the outputs derived from it, each of the last three NULL when not wanted: the xpgk
// (From<&ExtendedSpendingKey>: the same header, key = sk P_G), dk and ek.  The three cost one fixed-base product for pgk
// when any is wanted, and one more for ek.
ZK_DEV void hd_put_xsk(uint32_t depth, uint32_t tag, uint32_t index, const uint32_t *chain, const Fs &sk, uint8_t *xsk, uint8_t *xpgk,
                       uint8_t *dk, uint8_t *ek) {
    hd_put(xsk, depth, tag, index, chain, sk.l);
    if (!xpgk && !dk && !ek) return;
    uint32_t pgk[8];
    ext_encode(pg_mul(sk), pgk);
    if (xpgk) hd_put(xpgk, depth, tag, index, chain, pgk);
    if (dk || ek) hd_dk_ek(pgk, dk, ek);
}

// ---- rows -------------------------------------------------------------------------------------------------------------------
// one row of zk_xsk_master_batch
ZK_DEV void xsk_master(const uint8_t *seed, uint64_t len, uint8_t *xsk, uint8_t *xpgk, uint8_t *dk, uint8_t *ek) {
    uint32_t chain[8];
    const Fs sk = hd_master(seed, len, chain);
    hd_put_xsk(0, 0, 0, chain, sk, xsk, xpgk, dk, ek);
}

// The parent pass of zk_xsk_derive_batch for one named parent (73 bytes): false when its sk >= r_J (SpendingKey::read
// fails); otherwise pgk = Point::write(sk P_G) and tag = its EncKeyTag
ZK_DEV bool xsk_parent(const uint8_t *parent, uint32_t *pgk, uint32_t &tag) {
    uint32_t sk[8];
    hd_load(parent + HD_KEY, sk);
    if (!Fs::canonical_lt_mod(fs_words(sk))) return false;
    ext_encode(pg_mul(fs_words(sk)), pgk);
    tag = hd_tag(pgk);
    return true;
}
// ExtendedSpendingKey::derive_child(index) of a parent (73 bytes, sk < r_J, depth < 255) whose pgk encoding and tag
// xsk_parent gave; outputs as hd_put_xsk
ZK_DEV void xsk_child(const uint8_t *parent, const uint32_t *pgk, uint32_t tag, uint32_t index, uint8_t *xsk, uint8_t *xpgk, uint8_t *dk,
                      uint8_t *ek) {
    uint32_t c[8], sk[8], key[8], chain[8];
    hd_load(parent + HD_CHAIN, c);
    hd_load(parent + HD_KEY, sk);
    const bool hard = index >= HD_HARDENED_BIT;
#pragma unroll
    for (int i = 0; i < 8; i++) key[i] = hard ? sk[i] : pgk[i];
    uint64_t I[8];
    hd_prf_child(c, hard ? 0x11u : 0x12u, key, index, I);
#pragma unroll
    for (int i = 0; i < 4; i++) { chain[2 * i] = (uint32_t)I[4 + i]; chain[2 * i + 1] = (uint32_t)(I[4 + i] >> 32); }
    hd_put_xsk(parent[0] + 1u, tag, index, chain, hd_tweak(I) + fs_words(sk), xsk, xpgk, dk, ek);
}

// The parent pass of zk_xpgk_derive_batch for one named parent (73 bytes): ProofGenerationKey::read of its key, returning
// the zk_jubjub_into_xy status.  On JJ_OK: pgk = Point::write of the point read (the reference hashes the re-encoded
// point; it differs from the bytes only for the identity written with its sign bit set), niels its Niels form
// (TB_ENTRY_WORDS words, the layout load_niels reads) and tag its EncKeyTag.
ZK_DEV int xpgk_parent(const uint8_t *parent, uint32_t *pgk, uint32_t *niels, uint32_t &tag) {
    uint32_t w[8];
    hd_load(parent + HD_KEY, w);
    Ext p;
    const int st = read_prime_order(w, p);
    if (st != JJ_OK) return st;
    jubjub_encode(p.x, p.y, pgk);                 // jubjub_read leaves Z = 1
    const Niels q = niels_of(p.x, p.y, jj_d2());
#pragma unroll
    for (int i = 0; i < 8; i++) { niels[i] = q.ymx.l[i]; niels[8 + i] = q.ypx.l[i]; niels[16 + i] = q.kt.l[i]; }
    tag = hd_tag(pgk);
    return JJ_OK;
}
// ExtendedProofGenerationKey::derive_child(index) of a parent (73 bytes, a pgk of prime order, depth < 255, index < 2^31)
// whose pgk encoding, Niels form and tag xpgk_parent gave; dk and ek may be NULL
ZK_DEV void xpgk_child(const uint8_t *parent, const uint32_t *pgk, const Niels &q, uint32_t tag, uint32_t index, uint8_t *xpgk, uint8_t *dk,
                       uint8_t *ek) {
    uint32_t c[8], chain[8], child[8];
    hd_load(parent + HD_CHAIN, c);
    uint64_t I[8];
    hd_prf_child(c, 0x12u, pgk, index, I);
#pragma unroll
    for (int i = 0; i < 4; i++) { chain[2 * i] = (uint32_t)I[4 + i]; chain[2 * i + 1] = (uint32_t)(I[4 + i] >> 32); }
    ext_encode(ext_madd(pg_mul(hd_tweak(I)), q), child);
    hd_put(xpgk, parent[0] + 1u, tag, index, chain, child);
    if (dk || ek) hd_dk_ek(child, dk, ek);
}


// One row of zk_xsk_derive_batch after the parent pass: parent p (parents: n_parents extended keys) has pstatus[p] (0, or
// 1 for an sk >= r_J), and on 0 its pgk encoding at penc + 8 p and tag at ptag[p].  Returns the row's status, or -1 when
// the parent's sk >= r_J and the row is left unwritten: HD_BAD_INDEX for p >= n_parents, HD_DEPTH for a parent at depth
// 255 (the row's outputs zeroed), else 0.
ZK_DEV int xsk_row(const uint8_t *parents, size_t n_parents, uint32_t p, uint32_t index, const uint32_t *penc, const uint32_t *ptag,
                   const uint8_t *pstatus, uint8_t *xsk, uint8_t *xpgk, uint8_t *dk, uint8_t *ek) {
    if (p < n_parents && pstatus[p]) return -1;
    const uint8_t *parent = parents + (size_t)HD_XK_BYTES * (p < n_parents ? p : 0);
    const int st = p >= n_parents ? HD_BAD_INDEX : parent[0] > HD_MAX_DEPTH ? HD_DEPTH : JJ_OK;
    if (st != JJ_OK) {
        hd_zero(xsk, HD_XK_BYTES); hd_zero(xpgk, HD_XK_BYTES); hd_zero(dk, 32); hd_zero(ek, 32);
        return st;
    }
    uint32_t pgk[8];
#pragma unroll
    for (int k = 0; k < 8; k++) pgk[k] = penc[8 * (size_t)p + k];
    xsk_child(parent, pgk, ptag[p], index, xsk, xpgk, dk, ek);
    return JJ_OK;
}

// One row of zk_xpgk_derive_batch after the parent pass (pstatus[p]: xpgk_parent's status; on 0 the pgk encoding, tag and
// Niels form at penc + 8 p, ptag[p] and pniels + TB_ENTRY_WORDS p).  Returns the row's status: HD_BAD_INDEX for
// p >= n_parents, else the parent's read status, else HD_HARDENED for index >= 2^31, else HD_DEPTH for a parent at depth
// 255, else 0.  A row with a non-zero status has its outputs zeroed.
ZK_DEV int xpgk_row(const uint8_t *parents, size_t n_parents, uint32_t p, uint32_t index, const uint32_t *penc, const uint32_t *ptag,
                    const uint32_t *pniels, const uint8_t *pstatus, uint8_t *xpgk, uint8_t *dk, uint8_t *ek) {
    const uint8_t *parent = parents + (size_t)HD_XK_BYTES * (p < n_parents ? p : 0);
    const int st = p >= n_parents ? HD_BAD_INDEX : pstatus[p] != JJ_OK ? pstatus[p] : index >= HD_HARDENED_BIT ? HD_HARDENED
                   : parent[0] > HD_MAX_DEPTH ? HD_DEPTH : JJ_OK;
    if (st != JJ_OK) {
        hd_zero(xpgk, HD_XK_BYTES); hd_zero(dk, 32); hd_zero(ek, 32);
        return st;
    }
    uint32_t pgk[8];
#pragma unroll
    for (int k = 0; k < 8; k++) pgk[k] = penc[8 * (size_t)p + k];
    xpgk_child(parent, pgk, load_niels(pniels + TB_ENTRY_WORDS * (size_t)p), ptag[p], index, xpgk, dk, ek);
    return JJ_OK;
}

}  // namespace zkhd
