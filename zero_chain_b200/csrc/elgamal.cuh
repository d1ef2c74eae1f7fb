// Lifted-ElGamal balance decryption with the Diversifier generator: what zface's BalanceQuery runs before every transfer.
//
// Restates, value for value, DecryptionKey::read + Ciphertext::read (balance and pending transfer) + Ciphertext::add +
// Ciphertext::decrypt(dk, FixedGenerators::Diversifier) (core/keys/src/lib.rs:125-132, core/crypto/src/elgamal.rs:87-136,
// zface/src/utils/getter.rs:135-175):
//   dk              32 bytes, the Fs value little-endian; >= r_J is NotInField
//   Ciphertext      left | right, each Point::read + as_prime_order ([r_J] P == O)
//   V               (left + pending.left) - dk (right + pending.right)
//   decrypt         the i < 1 000 000 with i P_G == V, else None; the reference walks acc = O, P_G, 2 P_G, ... and compares
//                   whole points, so -i P_G (same y, other sign of x) is None
// The walk becomes a lookup: a table of the 10^6 canonical encodings of i P_G (y with the parity of x in bit 255, so the
// sign takes part in the comparison) and an open-addressing index over it.  Both are built once on the device:
//   eg_table_chunk    one thread per EG_CHUNK consecutive i: (i0) P_G by a 20-bit double-and-add, EG_CHUNK - 1 mixed
//                     additions of P_G, then one inversion for the whole chunk (Montgomery's trick) and the encodings
//   eg_index_insert   one thread per entry: slot = low bits of the encoding's first word, linear probing with a
//                     compare-and-swap; the slot holds a 12-bit fingerprint and i
// The entries are distinct points, so the order of insertion cannot change what a lookup finds.  A lookup accepts a slot
// only after comparing all 32 bytes of the table entry it names.
//
// Everything is inlined into the kernels (elgamal.cu) like jubjub.cuh and redjubjub.cuh; the table build and the index go
// through global memory only, so nothing goes to local memory.  The same source compiles with ZK_HOST_EMUL for the CPU test
// (tests/host_emul/emul_elgamal.cpp).
#pragma once
#include <stddef.h>
#include "redjubjub.cuh"

namespace zkeg {
using namespace zkjj;
using zkrj::Fs;
using zkrj::Niels;
using zkrj::ext_madd;
using zkrj::niels_identity;
using zkrj::niels_of;
using zkrj::niels_select;

enum Status : uint8_t { EG_OK = 0, EG_NOT_FOUND = 1, EG_BAD_KEY = 2, EG_BAD_BALANCE = 3, EG_BAD_PENDING = 4 };

constexpr uint32_t EG_BOUND = 1000000;         // elgamal.rs:102
constexpr uint32_t EG_CHUNK = 16;              // table entries per thread of the build
constexpr int EG_INDEX_LOG = 21;               // 2^21 slots for 10^6 entries: load factor 0.48
constexpr uint32_t EG_INDEX_MASK = (1u << EG_INDEX_LOG) - 1;
constexpr uint32_t EG_EMPTY = 0xffffffffu;     // never a valid slot: its entry bits would be 2^20 - 1 >= EG_BOUND
constexpr int EG_ENTRY_BITS = 20;              // slot = fingerprint << 20 | i
static_assert(EG_BOUND < (1u << EG_ENTRY_BITS), "entry numbers must fit below the fingerprint");

// P_G as a Niels point: the negation of RJ_NEG_PG swaps y - x and y + x and negates 2d x y
ZK_DEV Niels niels_pg() {
    Niels q;
#pragma unroll
    for (int i = 0; i < 8; i++) { q.ymx.l[i] = zkrj::RJ_NEG_PG[1][i]; q.ypx.l[i] = zkrj::RJ_NEG_PG[0][i]; q.kt.l[i] = zkrj::RJ_NEG_PG[2][i]; }
    q.kt = q.kt.neg();
    return q;
}

ZK_DEV void fr_store(uint32_t *dst, const Fr &a) {
#pragma unroll
    for (int i = 0; i < 8; i++) dst[i] = a.l[i];
}
ZK_DEV Fr fr_load(const uint32_t *src) {
    Fr a;
#pragma unroll
    for (int i = 0; i < 8; i++) a.l[i] = src[i];
    return a;
}

// ---- the table ---------------------------------------------------------------------------------------------------------
// Entries [t EG_CHUNK, min((t + 1) EG_CHUNK, n)) of the table: the encoding of i P_G in table[8 i .. 8 i + 8).  scratch
// holds 24 words per entry (X, Y, Z).  The forward pass keeps the running product of the Z's in the entry's table slot; the
// backward pass turns it into each Z's inverse and overwrites the slot with the encoding.  n <= 2^20.
ZK_DEV void eg_table_chunk(uint32_t t, uint32_t n, uint32_t *scratch, uint32_t *table) {
    const uint32_t i0 = t * EG_CHUNK;
    if (i0 >= n) return;
    const uint32_t cnt = n - i0 < EG_CHUNK ? n - i0 : EG_CHUNK;
    const Niels pg = niels_pg();
    Ext p = ext_identity();
#pragma unroll 1
    for (int b = EG_ENTRY_BITS - 1; b >= 0; b--) {      // (i0) P_G, the addend picked without a branch
        p = ext_dbl(p);
        p = ext_madd(p, niels_select((i0 >> b) & 1u, pg, niels_identity()));
    }
    Fr c = Fr::one();
#pragma unroll 1
    for (uint32_t j = 0; j < cnt; j++) {
        if (j) p = ext_madd(p, pg);
        uint32_t *s = scratch + 24 * (size_t)(i0 + j);
        fr_store(s, p.x); fr_store(s + 8, p.y); fr_store(s + 16, p.z);
        c = c * p.z;
        fr_store(table + 8 * (size_t)(i0 + j), c);        // Z_0 ... Z_j
    }
    Fr inv = c.inverse();                                 // (Z_0 ... Z_{cnt-1})^-1
#pragma unroll 1
    for (uint32_t j = cnt; j-- > 0;) {
        const size_t i = i0 + j;
        const uint32_t *s = scratch + 24 * i;
        const Fr zi = j ? fr_load(table + 8 * (i - 1)) * inv : inv;   // Z_j^-1
        inv = inv * fr_load(s + 16);                                     // (Z_0 ... Z_{j-1})^-1
        jubjub_encode(fr_load(s) * zi, fr_load(s + 8) * zi, table + 8 * i);
    }
}

// ---- the index ---------------------------------------------------------------------------------------------------------
ZK_DEV uint32_t eg_fingerprint(const uint32_t *enc) { return enc[1] >> EG_ENTRY_BITS; }   // 12 bits, disjoint from the slot bits

ZK_DEV uint32_t eg_cas(uint32_t *a, uint32_t expect, uint32_t val) {
#ifdef ZK_HOST_EMUL
    const uint32_t old = *a;
    if (old == expect) *a = val;
    return old;
#else
    return atomicCAS(a, expect, val);
#endif
}

// Inserts entry i with encoding enc.  The index (mask + 1 slots, all EG_EMPTY to begin with) must have a free slot.
ZK_DEV void eg_index_insert(uint32_t *index, uint32_t mask, const uint32_t *enc, uint32_t i) {
    const uint32_t v = (eg_fingerprint(enc) << EG_ENTRY_BITS) | i;
    for (uint32_t h = enc[0] & mask;; h = (h + 1) & mask)
        if (eg_cas(index + h, EG_EMPTY, v) == EG_EMPTY) return;
}

// The entry whose 32-byte table encoding equals enc, or EG_EMPTY.  A matching fingerprint only sends the probe to the table.
ZK_DEV uint32_t eg_lookup(const uint32_t *index, uint32_t mask, const uint32_t *table, const uint32_t *enc) {
    const uint32_t fp = eg_fingerprint(enc);
    for (uint32_t h = enc[0] & mask;; h = (h + 1) & mask) {
        const uint32_t v = index[h];
        if (v == EG_EMPTY) return EG_EMPTY;
        if (v >> EG_ENTRY_BITS != fp) continue;
        const uint32_t i = v & ((1u << EG_ENTRY_BITS) - 1);
        const uint32_t *e = table + 8 * (size_t)i;
        uint32_t diff = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) diff |= e[k] ^ enc[k];
        if (!diff) return i;
    }
}

// ---- one ciphertext ----------------------------------------------------------------------------------------------------
ZK_DEV Ext ext_select(bool c, const Ext &a, const Ext &b) {   // c ? a : b, without a branch
    Ext r;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.x.l[i] = c ? a.x.l[i] : b.x.l[i];
        r.y.l[i] = c ? a.y.l[i] : b.y.l[i];
        r.z.l[i] = c ? a.z.l[i] : b.z.l[i];
        r.t.l[i] = c ? a.t.l[i] : b.t.l[i];
    }
    return r;
}
// Point::read + as_prime_order
ZK_DEV bool eg_read_prime_order(const uint32_t *enc, Ext &p) {
    return jubjub_read(enc, p) == JJ_OK && ext_is_identity(ext_mul_order(p, jj_d2()));
}

// 32 little-endian bytes as 8 words (byte loads: a device pointer passed in by the caller need not be word aligned)
ZK_DEV void load_le_words(const uint8_t *b, uint32_t *w) {
#pragma unroll
    for (int i = 0; i < 8; i++)
        w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
}

// Everything of one decryption but the lookup.  dk: 32 bytes; ct, pend: 64 (left then right); pend NULL: no pending
// transfer.  The bytes are read where they are used, so no more than one point's words are live at a time.  Returns
// EG_BAD_KEY / EG_BAD_BALANCE / EG_BAD_PENDING, the first in zface's order, or EG_OK with the encoding of
// V = left - dk right in venc.
ZK_DEV int elgamal_stage(const uint8_t *dk, const uint8_t *ct, const uint8_t *pend, uint32_t *venc) {
    uint32_t w[8];
    {
        Fs s;
        load_le_words(dk, w);
#pragma unroll
        for (int i = 0; i < 8; i++) s.l[i] = w[i];
        if (!Fs::canonical_lt_mod(s)) return EG_BAD_KEY;
    }
    // the balance's left and right points, then the pending transfer's, read one after the other by the same code and
    // summed into l and r
    const Fr d2 = jj_d2();
    Ext l = ext_identity(), r = ext_identity();
    const int n_points = pend ? 4 : 2;
#pragma unroll 1
    for (int k = 0; k < n_points; k++) {
        uint32_t e[8];
        load_le_words(k < 2 ? ct + 32 * k : pend + 32 * (k - 2), e);
        Ext p;
        if (!eg_read_prime_order(e, p)) return k < 2 ? EG_BAD_BALANCE : EG_BAD_PENDING;
        const bool left = (k & 1) == 0;
        const Ext s = ext_add(ext_select(left, l, r), p, d2);
        l = ext_select(left, s, l);
        r = ext_select(left, r, s);
    }
    Niels nr;                                             // -right, made affine
    {
        const Fr zi = r.z.inverse();
        nr = niels_of((r.x * zi).neg(), r.y * zi, d2);
    }
    // dk < r_J < 2^252: shift bit 251 up to bit 255, then take the top bit of each step
    load_le_words(dk, w);
#pragma unroll
    for (int i = 7; i > 0; i--) w[i] = (w[i] << 4) | (w[i - 1] >> 28);
    w[0] <<= 4;
    Ext acc = ext_identity();
#pragma unroll 1
    for (int i = 0; i < 252; i++) {
        if (i) acc = ext_dbl(acc);
        const bool b = w[7] >> 31;
        zkrj::shl1(w);
        acc = ext_madd(acc, niels_select(b, nr, niels_identity()));
    }
    const Ext v = ext_add(l, acc, d2);
    const Fr zi = v.z.inverse();
    jubjub_encode(v.x * zi, v.y * zi, venc);
    return EG_OK;
}

// Ciphertext::decrypt for one ciphertext against the table: the status, and the amount when it is EG_OK (else 0)
ZK_DEV int elgamal_decrypt(const uint8_t *dk, const uint8_t *ct, const uint8_t *pend, const uint32_t *table,
                           const uint32_t *index, uint32_t mask, uint32_t &value) {
    uint32_t enc[8];
    value = 0;
    const int st = elgamal_stage(dk, ct, pend, enc);
    if (st != EG_OK) return st;
    const uint32_t i = eg_lookup(index, mask, table, enc);
    if (i == EG_EMPTY) return EG_NOT_FOUND;
    value = i;
    return EG_OK;
}

}  // namespace zkeg
