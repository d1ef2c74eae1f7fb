// The sender side of a confidential transfer: key derivation, GEpoch::group_hash, the transfer's ElGamal ciphertexts with
// rvk and nonce, and RedJubjub signing, all with the Diversifier generator P_G.  Restates, value for value:
//   SpendingKey::from_seed    to_uniform(BLAKE2b-512 "zech_ExpandSeed_" (seed))            core/keys/src/lib.rs:64-71
//   ProofGenerationKey        sk P_G
//   into_decryption_key       BLAKE2s-256 "zech_bdk" (Point::write(pgk)), h[31] &= 7         lib.rs:181-199
//   EncryptionKey             dk P_G
//   GEpoch::group_hash(e)     the first tag byte i in 0..254 with [8] Point::read(BLAKE2s-256 "zcgepoch"
//                             (GH_FIRST_BLOCK || e as u32 LE || i)) != O; the reference asserts before tag 255
//                             core/primitives/src/g_epoch.rs:102-145, core/jubjub/src/group_hash.rs:17-45
//   Ciphertext::encrypt       (amount P_G + r ek, r P_G)                                      core/crypto/src/elgamal.rs:48-66
//   rvk, rsk                  pgk + alpha P_G, sk + alpha                                     lib.rs:167-177, redjubjub.rs:58-62
//   nonce                     dk g_epoch                                                      core/proofs/src/confidential.rs:131
//   PrivateKey::sign          r = H*(T || M), R = r P_G, S = r + H*(Rbar || M) sk             redjubjub.rs:73-103
//   the anonymous transfer    neg_encrypt / encrypt / encrypt(0) in gen_proof's ring order     core/proofs/src/anonymous.rs:97-145
//
// Every multiple of P_G goes through one fixed-base multiplication: signed 4-bit digits (63 windows of a scalar < 2^252
// and a carry window), one mixed addition per window from the table d 16^j P_G, d <= 8 (pg_table.inc, global memory,
// 96 B per entry), 64 additions = 448 Fr products; a 32-bit scalar takes 9 windows = 63 products.  The multiples of one
// g_epoch use the same code on a table built once per call (tb_epoch_entry).  Because ek_sender = dk P_G and
// rvk = (sk + alpha) P_G lie in the prime-order group, r ek_sender = (r dk) P_G, amount P_G + r ek_sender =
// (amount + r dk) P_G and pgk + alpha P_G = rsk P_G: the same points from one fixed-base multiplication each.  Only
// r ek_recipient needs a variable base: a 252-step double-and-add that adds the base or the identity, picked without a
// branch (~3.8 k products).
//
// Everything is inlined into the kernels (tx_build.cu).  Thread-local arrays are only indexed with compile-time constants:
// the hash rounds are unrolled, scalar digits are shifted out of the low word, and the window tables are read from global
// memory.  The same source compiles with ZK_HOST_EMUL for the CPU test (tests/host_emul/emul_tx_build.cpp).
#pragma once
#include <stddef.h>
#include "redjubjub.cuh"

namespace zktb {
using namespace zkrj;

#ifdef ZK_HOST_EMUL
#define ZK_TB_TABLE static const
#else
#define ZK_TB_TABLE static __device__ __align__(16) const
#endif
#include "pg_table.inc"

constexpr int TB_WINDOWS = 64, TB_DIGITS = 9, TB_ENTRY_WORDS = 24;
constexpr int TB_TABLE_WORDS = TB_WINDOWS * TB_DIGITS * TB_ENTRY_WORDS;
constexpr int TB_N_FIELDS = 9;    // 32-byte points per confidential_fields row (tx_build.cu)
constexpr int TB_MAX_TAG = 255;   // group_hash: tag bytes 0..254; g_epoch.rs asserts before 255

// ---- BLAKE2s-256 (RFC 7693) with an empty key and salt and an 8-byte personalization -----------------------------------
ZK_DEV constexpr uint32_t b2s_iv(int i) {
    constexpr uint32_t v[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    return v[i];
}
// "zech_bdk" (core/keys/src/lib.rs:41) and "zcgepoch" (g_epoch.rs:18) as two little-endian words
constexpr uint32_t TB_BDK0 = 0x6863657au, TB_BDK1 = 0x6b64625fu, TB_GEPOCH0 = 0x6567637au, TB_GEPOCH1 = 0x68636f70u;
// "zech_ExpandSeed_" (lib.rs:40) as two little-endian words
constexpr uint64_t TB_EXPAND0 = 0x7078455f6863657aull, TB_EXPAND1 = 0x5f64656553646e61ull;
// GH_FIRST_BLOCK (core/jubjub/src/constants.rs:5-6), 64 ASCII bytes, as 16 little-endian words
ZK_DEV constexpr uint32_t gh_first_block(int i) {
    constexpr uint32_t v[16] = {0x62363930u, 0x35613633u, 0x62343038u, 0x65636166u, 0x39363166u, 0x37316531u, 0x36336333u, 0x37346136u,
                                0x62356666u, 0x61343861u, 0x32663434u, 0x64646436u, 0x64386537u, 0x39376639u, 0x34623564u, 0x30666432u};
    return v[i];
}

ZK_DEV uint32_t rotr32(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
ZK_DEV void b2s_g(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t &d, uint32_t x, uint32_t y) {
    a = a + b + x; d = rotr32(d ^ a, 16); c = c + d; b = rotr32(b ^ c, 12);
    a = a + b + y; d = rotr32(d ^ a, 8); c = c + d; b = rotr32(b ^ c, 7);
}
// F(h, m, t, last): all 10 rounds unrolled (BLAKE2s uses BLAKE2b's first ten permutations)
ZK_DEV void b2s_compress(uint32_t *h, const uint32_t *m, uint32_t t, bool last) {
    uint32_t v[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { v[i] = h[i]; v[i + 8] = b2s_iv(i); }
    v[12] ^= t;                                   // the high word of the counter stays 0
    if (last) v[14] = ~v[14];
#pragma unroll
    for (int r = 0; r < 10; r++) {
        b2s_g(v[0], v[4], v[8], v[12], m[b2b_sigma(r, 0)], m[b2b_sigma(r, 1)]);
        b2s_g(v[1], v[5], v[9], v[13], m[b2b_sigma(r, 2)], m[b2b_sigma(r, 3)]);
        b2s_g(v[2], v[6], v[10], v[14], m[b2b_sigma(r, 4)], m[b2b_sigma(r, 5)]);
        b2s_g(v[3], v[7], v[11], v[15], m[b2b_sigma(r, 6)], m[b2b_sigma(r, 7)]);
        b2s_g(v[0], v[5], v[10], v[15], m[b2b_sigma(r, 8)], m[b2b_sigma(r, 9)]);
        b2s_g(v[1], v[6], v[11], v[12], m[b2b_sigma(r, 10)], m[b2b_sigma(r, 11)]);
        b2s_g(v[2], v[7], v[8], v[13], m[b2b_sigma(r, 12)], m[b2b_sigma(r, 13)]);
        b2s_g(v[3], v[4], v[9], v[14], m[b2b_sigma(r, 14)], m[b2b_sigma(r, 15)]);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}
// The 32-byte digest of a len-byte message whose k-th little-endian word is word(k) (zero past the end).  Both device
// callers pass a constant len, so the block loop unrolls and word() is called with constants.
template <class Word>
ZK_DEV void b2s_256(uint32_t pers0, uint32_t pers1, uint32_t len, Word word, uint32_t *h) {
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = b2s_iv(i);
    h[0] ^= 0x01010020u;                          // digest length 32, key length 0, fanout 1, depth 1
    h[6] ^= pers0;
    h[7] ^= pers1;
    const uint32_t nblocks = len ? (len + 63) / 64 : 1;
#pragma unroll
    for (uint32_t b = 0; b < nblocks; b++) {
        uint32_t m[16];
#pragma unroll
        for (int w = 0; w < 16; w++) m[w] = word(16 * b + w);
        const bool last = b + 1 == nblocks;
        b2s_compress(h, m, last ? len : 64 * (b + 1), last);
    }
}

// ---- BLAKE2b-512 of P prefix words || msg, with a 16-byte personalization ------------------------------------------------
template <int P>
ZK_DEV void b2b_prefixed(uint64_t pers0, uint64_t pers1, const uint64_t *pre, const uint8_t *msg, uint64_t mlen, uint64_t *h) {
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = b2b_iv(i);
    h[0] ^= 0x01010040ull;
    h[6] ^= pers0;
    h[7] ^= pers1;
    const uint64_t len = 8 * P + mlen, nblocks = len ? (len + 127) / 128 : 1;
    for (uint64_t b = 0; b < nblocks; b++) {
        uint64_t m[16];
#pragma unroll
        for (int w = 0; w < 16; w++) m[w] = (b == 0 && w < P) ? pre[w < P ? w : 0] : msg_word(msg, mlen, 128 * b + 8 * w - 8 * P);
        const bool last = b + 1 == nblocks;
        b2b_compress(h, m, last ? len : 128 * (b + 1), last);
    }
}

// ---- Fs helpers: canonical little-endian words in, canonical out ---------------------------------------------------------
ZK_DEV Fs fs_words(const uint32_t *w) {
    Fs r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.l[i] = w[i];
    return r;
}
ZK_DEV Fs fs_mul(const Fs &a, const Fs &b) { return a * Fs::from_canonical(b); }   // a b mod r_J, canonical
ZK_DEV Fs fs_u32(uint32_t v) { Fs r = Fs::zero(); r.l[0] = v; return r; }

// ---- fixed-base multiplication ------------------------------------------------------------------------------------------
ZK_DEV Niels load_niels(const uint32_t *p) {
    Niels q;
#ifdef ZK_HOST_EMUL
    for (int i = 0; i < 8; i++) { q.ymx.l[i] = p[i]; q.ypx.l[i] = p[8 + i]; q.kt.l[i] = p[16 + i]; }
#else
    const uint4 *v = reinterpret_cast<const uint4 *>(p);    // entries are 96 B, tables 16-byte aligned
    uint4 w[6];
#pragma unroll
    for (int i = 0; i < 6; i++) w[i] = __ldg(v + i);
#pragma unroll
    for (int i = 0; i < 2; i++) {
        q.ymx.l[4 * i] = w[i].x; q.ymx.l[4 * i + 1] = w[i].y; q.ymx.l[4 * i + 2] = w[i].z; q.ymx.l[4 * i + 3] = w[i].w;
        q.ypx.l[4 * i] = w[2 + i].x; q.ypx.l[4 * i + 1] = w[2 + i].y; q.ypx.l[4 * i + 2] = w[2 + i].z; q.ypx.l[4 * i + 3] = w[2 + i].w;
        q.kt.l[4 * i] = w[4 + i].x; q.kt.l[4 * i + 1] = w[4 + i].y; q.kt.l[4 * i + 2] = w[4 + i].z; q.kt.l[4 * i + 3] = w[4 + i].w;
    }
#endif
    return q;
}
ZK_DEV Niels niels_cneg(bool c, const Niels &a) {   // -(x, y) = (-x, y): y - x and y + x swap, 2d x y changes sign
    Niels r;
    const Fr nk = a.kt.neg();
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.ymx.l[i] = c ? a.ypx.l[i] : a.ymx.l[i];
        r.ypx.l[i] = c ? a.ymx.l[i] : a.ypx.l[i];
        r.kt.l[i] = c ? nk.l[i] : a.kt.l[i];
    }
    return r;
}
ZK_DEV void shr4(uint32_t *w) {
#pragma unroll
    for (int i = 0; i < 7; i++) w[i] = (w[i] >> 4) | (w[i + 1] << 28);
    w[7] >>= 4;
}
// acc + k T for a scalar k < 2^(4 NW - 4) (8 little-endian words) and a window table T of TB_WINDOWS x TB_DIGITS
// entries: digit j = window j + carry, taken as digit - 16 with a carry out when it exceeds 8.  NW = 64 covers k < 2^252,
// NW = 9 a 32-bit k.
template <int NW>
ZK_DEV Ext fb_mul(const uint32_t *__restrict__ table, const uint32_t *k, Ext acc = ext_identity()) {
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = k[i];
    uint32_t carry = 0;
#pragma unroll 1
    for (int j = 0; j < NW; j++) {
        const uint32_t v = (w[0] & 15u) + carry;
        shr4(w);
        const bool neg = v > 8;
        carry = neg;
        const Niels q = load_niels(table + (size_t)(TB_DIGITS * j + (neg ? 16 - v : v)) * TB_ENTRY_WORDS);
        acc = ext_madd(acc, niels_cneg(neg, q));
    }
    return acc;
}
ZK_DEV Ext pg_mul(const Fs &k) { return fb_mul<TB_WINDOWS>(TB_PG_TABLE, k.l); }

// k P for an affine P and k < 2^252: MSB-first double-and-add, adding P or the identity
ZK_DEV Ext vb_mul(const Niels &p, const uint32_t *k) {
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = k[i];
#pragma unroll
    for (int i = 7; i > 0; i--) w[i] = (w[i] << 4) | (w[i - 1] >> 28);
    w[0] <<= 4;
    Ext acc = ext_identity();
#pragma unroll 1
    for (int i = 0; i < 252; i++) {
        if (i) acc = ext_dbl(acc);
        const bool b = w[7] >> 31;
        shl1(w);
        acc = ext_madd(acc, niels_select(b, p, niels_identity()));
    }
    return acc;
}

// entry e = TB_DIGITS j + d of the window table of g: d 16^j g, affine, in Niels form (one inversion)
ZK_DEV void tb_epoch_entry(const Ext &g, int e, uint32_t *out) {
    const Fr d2 = jj_d2();
    Ext b = g;
    for (int i = 0; i < 4 * (e / TB_DIGITS); i++) b = ext_dbl(b);
    const int d = e % TB_DIGITS;
    Ext acc = ext_identity();
    for (int bit = 3; bit >= 0; bit--) {
        acc = ext_dbl(acc);
        if ((d >> bit) & 1) acc = ext_add(acc, b, d2);
    }
    const Fr zi = acc.z.inverse();
    const Niels q = niels_of(acc.x * zi, acc.y * zi, d2);
#pragma unroll
    for (int i = 0; i < 8; i++) { out[i] = q.ymx.l[i]; out[8 + i] = q.ypx.l[i]; out[16 + i] = q.kt.l[i]; }
}

// Point::write of an extended point (one inversion)
ZK_DEV void ext_encode(const Ext &p, uint32_t *enc) {
    const Fr zi = p.z.inverse();
    jubjub_encode(p.x * zi, p.y * zi, enc);
}
// Point::read + as_prime_order; JJ_OK or the zk_jubjub_into_xy status
ZK_DEV int read_prime_order(const uint32_t *enc, Ext &p) {
    const int s = jubjub_read(enc, p);
    if (s != JJ_OK) return s;
    return ext_is_identity(ext_mul_order(p, jj_d2())) ? JJ_OK : JJ_NOT_PRIME_ORDER;
}

// ---- keys ---------------------------------------------------------------------------------------------------------------
ZK_DEV Fs spending_key(const uint8_t *seed, uint64_t len) {
    uint64_t h[8];
    b2b_prefixed<0>(TB_EXPAND0, TB_EXPAND1, nullptr, seed, len, h);
    return fs_to_uniform(h);
}
// into_decryption_key(sk P_G).  The mask leaves dk < 2^251 < r_J, so the reference's NotInField branch cannot occur.
ZK_DEV Fs decryption_key(const Fs &sk) {
    uint32_t pgk[8], h[8];
    ext_encode(pg_mul(sk), pgk);
    b2s_256(TB_BDK0, TB_BDK1, 32, [&](uint32_t k) { return k < 8 ? pgk[k & 7] : 0u; }, h);
    h[7] &= 0x07ffffffu;
    return fs_words(h);
}

// ---- GEpoch::group_hash -------------------------------------------------------------------------------------------------
// The encoding of GEpoch::group_hash(epoch) and the tag byte it took; false (enc unset) when no tag below 255 gives a point.
ZK_DEV bool g_epoch_hash(uint32_t epoch, uint32_t *enc, uint32_t &tag_out) {
#pragma unroll 1
    for (uint32_t tag = 0; tag < TB_MAX_TAG; tag++) {
        uint32_t h[8];
        b2s_256(TB_GEPOCH0, TB_GEPOCH1, 69, [&](uint32_t k) { return k < 16 ? gh_first_block(k & 15) : k == 16 ? epoch : k == 17 ? tag : 0u; }, h);
        Ext p;
        if (jubjub_read(h, p) != JJ_OK) continue;
        p = ext_dbl(ext_dbl(ext_dbl(p)));        // mul_by_cofactor
        if (ext_is_identity(p)) continue;
        ext_encode(p, enc);
        tag_out = tag;
        return true;
    }
    return false;
}

// ---- signing ------------------------------------------------------------------------------------------------------------
// PrivateKey::sign(msg, T) for sk < r_J: rbar || sbar as 16 little-endian words.  t: the 80 bytes of T as 10 words.
ZK_DEV void redjubjub_sign(const Fs &sk, const uint64_t *t, const uint8_t *msg, uint64_t mlen, uint32_t *sig) {
    uint64_t h[8];
    b2b_prefixed<10>(RJ_PERSONAL0, RJ_PERSONAL1, t, msg, mlen, h);
    const Fs r = fs_to_uniform(h);
    ext_encode(pg_mul(r), sig);
    uint64_t rbar[4];
#pragma unroll
    for (int i = 0; i < 4; i++) rbar[i] = (uint64_t)sig[2 * i] | ((uint64_t)sig[2 * i + 1] << 32);
    h_star_digest(rbar, msg, mlen, h);
    const Fs s = fs_mul(fs_to_uniform(h), sk) + r;
#pragma unroll
    for (int i = 0; i < 8; i++) sig[8 + i] = s.l[i];
}

// ---- the confidential transfer's fields ---------------------------------------------------------------------------------
ZK_DEV void store_le_words(uint8_t *b, const uint32_t *w, int n) {
#pragma unroll
    for (int i = 0; i < n; i++)     // byte stores: a device pointer passed in by the caller need not be word aligned
        for (int k = 0; k < 4; k++) b[4 * i + k] = (uint8_t)(w[i] >> (8 * k));
}
// scratch slot s (0 .. 27) of a row: 8 words at scratch[(8 s + w) stride]
ZK_DEV void tb_put(uint32_t *scratch, size_t stride, int s, const Fr &v) {
#pragma unroll
    for (int w = 0; w < 8; w++) scratch[(8 * (size_t)s + w) * stride] = v.l[w];
}
ZK_DEV Fr tb_get(const uint32_t *scratch, size_t stride, int s) {
    Fr v;
#pragma unroll
    for (int w = 0; w < 8; w++) v.l[w] = scratch[(8 * (size_t)s + w) * stride];
    return v;
}

// One row of zk_confidential_fields_batch.  sk, r, alpha < r_J and the g_epoch encoding g_enc with its window table are
// the caller's to check.  fields: TB_N_FIELDS encodings in ConfidentialTx order (address_sender, address_recipient,
// amount_sender, amount_recipient, fee_sender, randomness, rvk, g_epoch, nonce); the seven computed points are made
// affine with one inversion, their X, Y, Z and Z-prefix products parked in scratch (28 slots) between the passes.  A
// recipient key that fails EncryptionKey::read zeroes the row and returns its zk_jubjub_into_xy status.
ZK_DEV int confidential_fields(const uint32_t *sk_w, const uint32_t *ekr_w, uint32_t amount, uint32_t fee, const uint32_t *r_w,
                               const uint32_t *alpha_w, const uint8_t *g_enc, const uint32_t *__restrict__ g_table, uint32_t *scratch,
                               size_t stride, uint8_t *fields, uint8_t *rsk_out, uint8_t *dk_out) {
    Ext ekr;
    const int st = read_prime_order(ekr_w, ekr);
    if (st != JJ_OK) {
        for (int i = 0; i < 32 * TB_N_FIELDS; i++) fields[i] = 0;
        for (int i = 0; i < 32; i++) rsk_out[i] = dk_out[i] = 0;
        return st;
    }
    store_le_words(fields + 32, ekr_w, 8);                    // address_recipient
    for (int i = 0; i < 32; i++) fields[7 * 32 + i] = g_enc[i];   // g_epoch
    const Fr d2 = jj_d2();
    const Fs sk = fs_words(sk_w), r = fs_words(r_w), rsk = sk + fs_words(alpha_w);
    const Fs dk = decryption_key(sk), rdk = fs_mul(r, dk);
    Fr acc = Fr::one();
    auto stash = [&](int k, const Ext &p) {
        tb_put(scratch, stride, 4 * k, p.x); tb_put(scratch, stride, 4 * k + 1, p.y);
        tb_put(scratch, stride, 4 * k + 2, p.z); tb_put(scratch, stride, 4 * k + 3, acc);
        acc = acc * p.z;
    };
    {
        const uint32_t aw[8] = {amount, 0, 0, 0, 0, 0, 0, 0};   // amount_recipient = r ek_r + amount P_G
        stash(0, fb_mul<9>(TB_PG_TABLE, aw, vb_mul(niels_of(ekr.x, ekr.y, d2), r.l)));
    }
    stash(1, pg_mul(dk));                                     // address_sender = ek_s
    stash(2, pg_mul(fs_u32(amount) + rdk));                   // amount_sender = amount P_G + r ek_s
    stash(3, pg_mul(fs_u32(fee) + rdk));                      // fee_sender = fee P_G + r ek_s
    stash(4, pg_mul(r));                                      // randomness = r P_G
    stash(5, pg_mul(rsk));                                    // rvk = pgk + alpha P_G
    stash(6, fb_mul<TB_WINDOWS>(g_table, dk.l));              // nonce = dk g_epoch
    Fr inv = acc.inverse();
#pragma unroll 1
    for (int k = 6; k >= 0; k--) {
        const Fr zi = inv * tb_get(scratch, stride, 4 * k + 3);
        inv = inv * tb_get(scratch, stride, 4 * k + 2);
        uint32_t enc[8];
        jubjub_encode(tb_get(scratch, stride, 4 * k) * zi, tb_get(scratch, stride, 4 * k + 1) * zi, enc);
        const int slot = k == 0 ? 3 : k == 1 ? 0 : k == 2 ? 2 : k + 1 + (k == 6);   // 3, 0, 2, 4, 5, 6, 8
        store_le_words(fields + 32 * slot, enc, 8);
    }
    store_le_words(rsk_out, rsk.l, 8);
    store_le_words(dk_out, dk.l, 8);
    return JJ_OK;
}

// ---- the anonymous transfer's fields ------------------------------------------------------------------------------------
// zk_anonymous_fields_batch (tx_build.cu) runs a row in two passes: anonymous_row (one thread per row) computes what the
// sender's keys give, the sender's slot of both arrays, right_ciphertext, rvk and nonce; anonymous_left (one thread per
// ring entry) computes r ek for the recipient and each decoy from the call's key table, decoded once per distinct key
// (anon_key_entry).  Restates MultiCiphertexts::<Anonymous>::encrypt (core/proofs/src/crypto_components.rs:168-216):
//   sender     neg_encrypt: -amount P_G + r ek_s = (r dk - amount) P_G, because ek_s = dk P_G    core/crypto/src/elgamal.rs:70-85
//   recipient  encrypt: amount P_G + r ek_t
//   decoys     encrypt(0): r ek_d
// and places the entries where gen_proof's two Vec::insert calls put them (core/proofs/src/anonymous.rs:118-145).
constexpr int TB_RING = 12;                       // ANONIMITY_SIZE
constexpr int TB_RING_IN = TB_RING - 1;           // ring indices per row: the recipient, then the ten decoys
constexpr int TB_N_ANON_FIELDS = 2 * TB_RING + 3; // enc_keys[12] | left_ciphertexts[12] | right_ciphertext | rvk | nonce
constexpr int TB_ANON_BAD_INDEX = 4, TB_ANON_BAD_POSITIONS = 5;

// The ring position of MultiEncKeys entry j (0: the recipient, 1 .. 10: the decoys in order) with the sender at s and the
// recipient at t (s != t, both < 12).  Inserting the sender at s and the recipient at t into the ten decoys, in either
// order gen_proof uses, leaves the decoys in their order on the ten other positions.
ZK_DEV int anon_position(int s, int t, int j) {
    if (j == 0) return t;
    const int lo = s < t ? s : t, hi = s < t ? t : s;
    int p = j - 1;
    p += p >= lo;
    p += p >= hi;
    return p;
}

// EncryptionKey::read (Point::read + as_prime_order) of one key of the call's table: its JJ status, and its Niels form in
// out (TB_ENTRY_WORDS words, the layout load_niels reads; the identity's when the read fails)
ZK_DEV int anon_key_entry(const uint32_t *enc, uint32_t *out) {
    Ext p;
    const int st = read_prime_order(enc, p);
    const Niels q = st == JJ_OK ? niels_of(p.x, p.y, jj_d2()) : niels_identity();
#pragma unroll
    for (int i = 0; i < 8; i++) { out[i] = q.ymx.l[i]; out[8 + i] = q.ypx.l[i]; out[16 + i] = q.kt.l[i]; }
    return st;
}

// A row's status: TB_ANON_BAD_POSITIONS for s >= 12, t >= 12 or s = t; else TB_ANON_BAD_INDEX for a ring index >= n_keys;
// else the zk_jubjub_into_xy code of the first key, in MultiEncKeys order, that fails EncryptionKey::read; else 0.
ZK_DEV int anon_status(int s, int t, const uint32_t *ring, size_t n_keys, const uint8_t *key_status) {
    if (s >= TB_RING || t >= TB_RING || s == t) return TB_ANON_BAD_POSITIONS;
#pragma unroll 1
    for (int j = 0; j < TB_RING_IN; j++)
        if (ring[j] >= n_keys) return TB_ANON_BAD_INDEX;
#pragma unroll 1
    for (int j = 0; j < TB_RING_IN; j++)
        if (key_status[ring[j]] != JJ_OK) return key_status[ring[j]];
    return JJ_OK;
}

// The row pass of one row: status from anon_status, sk / r / alpha < r_J, the sender at s.  A row with status 0 gets
// enc_keys[s] = ek_s, left_ciphertexts[s], right_ciphertext = r P_G, rvk = rsk P_G, nonce = dk g_epoch (g_table: the
// g_epoch's window table), rsk and dk; the five points are made affine with one inversion, their X, Y, Z and Z-prefix
// products parked in scratch (TB_ANON_SCRATCH_SLOTS slots) as in confidential_fields.  A row with another status gets
// zeros in all TB_N_ANON_FIELDS fields, rsk and dk, and anonymous_left leaves it alone.
constexpr int TB_ANON_SCRATCH_SLOTS = 20;
ZK_DEV void anonymous_row(int status, int s, const uint32_t *sk_w, uint32_t amount, const uint32_t *r_w, const uint32_t *alpha_w,
                          const uint32_t *__restrict__ g_table, uint32_t *scratch, size_t stride, uint8_t *fields, uint8_t *rsk_out,
                          uint8_t *dk_out) {
    if (status != JJ_OK) {
        for (int i = 0; i < 32 * TB_N_ANON_FIELDS; i++) fields[i] = 0;
        for (int i = 0; i < 32; i++) rsk_out[i] = dk_out[i] = 0;
        return;
    }
    const Fs sk = fs_words(sk_w), r = fs_words(r_w), rsk = sk + fs_words(alpha_w);
    const Fs dk = decryption_key(sk);
    Fr acc = Fr::one();
    auto stash = [&](int k, const Ext &p) {
        tb_put(scratch, stride, 4 * k, p.x); tb_put(scratch, stride, 4 * k + 1, p.y);
        tb_put(scratch, stride, 4 * k + 2, p.z); tb_put(scratch, stride, 4 * k + 3, acc);
        acc = acc * p.z;
    };
    stash(0, pg_mul(dk));                                     // enc_keys[s] = ek_s
    stash(1, pg_mul(fs_mul(r, dk) - fs_u32(amount)));         // left_ciphertexts[s] = -amount P_G + r ek_s
    stash(2, pg_mul(r));                                      // right_ciphertext = r P_G
    stash(3, pg_mul(rsk));                                    // rvk = pgk + alpha P_G
    stash(4, fb_mul<TB_WINDOWS>(g_table, dk.l));              // nonce = dk g_epoch
    Fr inv = acc.inverse();
#pragma unroll 1
    for (int k = 4; k >= 0; k--) {
        const Fr zi = inv * tb_get(scratch, stride, 4 * k + 3);
        inv = inv * tb_get(scratch, stride, 4 * k + 2);
        uint32_t enc[8];
        jubjub_encode(tb_get(scratch, stride, 4 * k) * zi, tb_get(scratch, stride, 4 * k + 1) * zi, enc);
        const int slot = k == 0 ? s : k == 1 ? TB_RING + s : 2 * TB_RING + k - 2;
        store_le_words(fields + 32 * slot, enc, 8);
    }
    store_le_words(rsk_out, rsk.l, 8);
    store_le_words(dk_out, dk.l, 8);
}

// Ring entry j of a row with status 0, at ring position p (anon_position): q is the entry's key in Niels form and key_enc
// its 32 table bytes, copied to enc_keys[p]; left_ciphertexts[p] = r key + amount P_G for the recipient (j = 0) and r key
// + 0 P_G for a decoy (the same 63 products in every lane of a warp, so no branch diverges).
ZK_DEV void anonymous_left(const Niels &q, const uint8_t *key_enc, int j, int p, uint32_t amount, const uint32_t *r_w, uint8_t *fields) {
    for (int i = 0; i < 32; i++) fields[32 * p + i] = key_enc[i];
    uint8_t *out = fields + 32 * (TB_RING + p);
    const uint32_t aw[8] = {j == 0 ? amount : 0u, 0, 0, 0, 0, 0, 0, 0};
    uint32_t enc[8];
    ext_encode(fb_mul<9>(TB_PG_TABLE, aw, vb_mul(q, r_w)), enc);
    store_le_words(out, enc, 8);
}

}  // namespace zktb
