/* TEST INFRASTRUCTURE (oracle) — zface's hierarchical key derivation (zface/src/derive/mod.rs) with the Diversifier generator,
 * in plain C99 + OpenMP.  Not part of the product; the tests and tools/hd_bench.py build it through
 * tests/jubjub_oracle/hd_coracle.py.
 *
 * It builds on the transaction-building oracle (tx_build_oracle.c, included as it is, which includes elgamal_oracle.c,
 * redjubjub_oracle.c and jubjub_oracle.c): BLAKE2b, BLAKE2s, Fs, SpendingKey::from_seed, into_decryption_key, P_G,
 * Point::read, Point::mul, Point::write.  Added here, each step the reference's way, every product its own double-and-add:
 *   master                   I = BLAKE2b-512 "Zerochain_Master" (seed), sk = SpendingKey::from_seed(I_L), chain code I_R
 *   xsk derive_child         prf_expand_vec(c, [0x11, sk, i] or [0x12, pgk, i]), sk' = to_uniform(prf_expand(I_L, [0x13]))
 *                            + sk, the tag from BLAKE2b-256 "ZerochainEFinger" (pgk)
 *   xpgk derive_child        pgk' = to_uniform(prf_expand(I_L, [0x13])) P_G + pgk; hardened indices refused
 *   From<&xsk>, dk, ek       sk' P_G, into_decryption_key(pgk'), dk P_G
 * in the layouts of zk_xsk_master_batch, zk_xsk_derive_batch and zk_xpgk_derive_batch.  Each row reads its own parent.
 * Rows are split over the OpenMP threads; it is the host-core baseline of the device calls. */
#include "tx_build_oracle.c"

static const uint8_t MASTER_PERSONAL[16] = {'Z', 'e', 'r', 'o', 'c', 'h', 'a', 'i', 'n', '_', 'M', 'a', 's', 't', 'e', 'r'};
static const uint8_t EKFP_PERSONAL[16] = {'Z', 'e', 'r', 'o', 'c', 'h', 'a', 'i', 'n', 'E', 'F', 'i', 'n', 'g', 'e', 'r'};
#define XK 73

/* prf_expand_vec(k, [a, b, c]) with a 64-byte digest (any part may be empty) */
static void prf_expand(uint8_t *out, const uint8_t *k, const uint8_t *a, size_t alen, const uint8_t *b, size_t blen, const uint8_t *c,
                       size_t clen) {
    b2b_t s;
    b2b_init(&s, EXPAND_SEED_PERSONAL);
    b2b_update(&s, k, 32);
    b2b_update(&s, a, alen); b2b_update(&s, b, blen); b2b_update(&s, c, clen);
    b2b_final(&s, out);
}
/* EncKeyFingerPrint::tag: the first 4 bytes of BLAKE2b-256 "ZerochainEFinger" (pgk); a 32-byte digest is the first half
 * of the final state of a hash whose parameter block says 32 */
static void ekfp_tag(uint8_t *tag, const uint8_t *pgk) {
    b2b_t s;
    uint8_t d[64];
    b2b_init(&s, EKFP_PERSONAL);
    s.h[0] = B2B_IV[0] ^ 0x01010020ULL;
    b2b_update(&s, pgk, 32);
    b2b_final(&s, d);
    memcpy(tag, d, 4);
}
static void put_u32(uint8_t *b, uint32_t v) { for (int k = 0; k < 4; k++) b[k] = (uint8_t)(v >> (8 * k)); }
static int fs_lt(const uint8_t *b) {   /* a 32-byte little-endian value < r_J */
    uint64_t w[4];
    load_le(w, b, 4);
    for (int i = 3; i >= 0; i--)
        if (w[i] != JJ_ORDER[i]) return w[i] < JJ_ORDER[i];
    return 0;
}
/* the account outputs of pgk (each may be NULL): the xpgk with xsk's header, dk and ek */
static void account(const uint8_t *hdr, const ext_t *pgk, uint8_t *xpgk, uint8_t *dkb, uint8_t *ekb) {
    uint8_t enc[32], h[32];
    ext_write(enc, pgk);
    if (xpgk) { memcpy(xpgk, hdr, 41); memcpy(xpgk + 41, enc, 32); }
    if (!dkb && !ekb) return;
    b2s_t s;
    b2s_init(&s, BDK_PERSONAL);
    b2s_update(&s, enc, 32);
    b2s_final(&s, h);
    h[31] &= 0x07;
    if (dkb) memcpy(dkb, h, 32);
    if (ekb) {
        uint64_t dk[4];
        ext_t ek;
        load_le(dk, h, 4);
        pg_mul(&ek, dk);
        ext_write(ekb, &ek);
    }
}

static void master(const uint8_t *seed, size_t len, uint8_t *xsk, uint8_t *xpgk, uint8_t *dkb, uint8_t *ekb) {
    b2b_t s;
    uint8_t i[64];
    uint64_t sk[4];
    b2b_init(&s, MASTER_PERSONAL);
    b2b_update(&s, seed, len);
    b2b_final(&s, i);
    spending_key(sk, i, 32);
    memset(xsk, 0, 9);
    memcpy(xsk + 9, i + 32, 32);
    store_le(xsk + 41, sk);
    ext_t pgk;
    pg_mul(&pgk, sk);
    account(xsk, &pgk, xpgk, dkb, ekb);
}

/* one row of zk_xsk_derive_batch (parent: NULL when out of range); its status */
static int xsk_child(const uint8_t *parent, uint32_t index, uint8_t *xsk, uint8_t *xpgk, uint8_t *dkb, uint8_t *ekb) {
    const int st = !parent ? 4 : parent[0] == 255 ? 6 : 0;
    if (st) {
        memset(xsk, 0, XK);
        if (xpgk) memset(xpgk, 0, XK);
        if (dkb) memset(dkb, 0, 32);
        if (ekb) memset(ekb, 0, 32);
        return st;
    }
    uint64_t sk[4], t[4];
    uint8_t enc[32], ib[4], h[64], th[64], one3 = 0x13, tag11 = 0x11, tag12 = 0x12;
    load_le(sk, parent + 41, 4);
    ext_t pgk, child;
    pg_mul(&pgk, sk);
    ext_write(enc, &pgk);
    put_u32(ib, index);
    if (index >> 31) prf_expand(h, parent + 9, &tag11, 1, parent + 41, 32, ib, 4);
    else prf_expand(h, parent + 9, &tag12, 1, enc, 32, ib, 4);
    prf_expand(th, h, &one3, 1, NULL, 0, NULL, 0);
    to_uniform(t, th);
    fs_t a, b;
    fs_from_repr(&a, t); fs_from_repr(&b, sk);
    fs_add(&a, &a, &b);
    fs_into_repr(t, &a);
    xsk[0] = (uint8_t)(parent[0] + 1);
    ekfp_tag(xsk + 1, enc);
    put_u32(xsk + 5, index);
    memcpy(xsk + 9, h + 32, 32);
    store_le(xsk + 41, t);
    if (!xpgk && !dkb && !ekb) return 0;
    pg_mul(&child, t);
    account(xsk, &child, xpgk, dkb, ekb);
    return 0;
}

/* one row of zk_xpgk_derive_batch (parent: NULL when out of range); its status */
static int xpgk_child(const uint8_t *parent, uint32_t index, uint8_t *xpgk, uint8_t *dkb, uint8_t *ekb) {
    ext_t pgk;
    int st = 4;
    if (parent) {
        st = read_point(parent + 41, &pgk);
        if (!st) {
            ext_t o;
            ext_mul(&o, &pgk, JJ_ORDER);
            if (!(fr_is_zero(&o.x) && fr_eq(&o.y, &o.z))) st = 3;
        }
        if (!st && (index >> 31)) st = 5;
        if (!st && parent[0] == 255) st = 6;
    }
    if (st) {
        memset(xpgk, 0, XK);
        if (dkb) memset(dkb, 0, 32);
        if (ekb) memset(ekb, 0, 32);
        return st;
    }
    uint64_t t[4];
    uint8_t enc[32], ib[4], h[64], th[64], one3 = 0x13, tag12 = 0x12, hdr[41];
    ext_write(enc, &pgk);
    put_u32(ib, index);
    prf_expand(h, parent + 9, &tag12, 1, enc, 32, ib, 4);
    prf_expand(th, h, &one3, 1, NULL, 0, NULL, 0);
    to_uniform(t, th);
    ext_t a, child;
    fr_t d2;
    jj_d2(&d2);
    pg_mul(&a, t);
    ext_add(&child, &a, &pgk, &d2);
    hdr[0] = (uint8_t)(parent[0] + 1);
    ekfp_tag(hdr + 1, enc);
    put_u32(hdr + 5, index);
    memcpy(hdr + 9, h + 32, 32);
    account(hdr, &child, xpgk, dkb, ekb);
    return 0;
}

EXPORT void hdo_tag(const uint8_t *pgk, uint8_t *tag) { ekfp_tag(tag, pgk); }
EXPORT void hdo_master(size_t n, const uint8_t *seeds, const uint64_t *off, uint8_t *xsks, uint8_t *xpgks, uint8_t *dks, uint8_t *eks) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < nn; i++)
        master(seeds + off[i], off[i + 1] - off[i], xsks + XK * i, xpgks ? xpgks + XK * i : NULL, dks ? dks + 32 * i : NULL,
               eks ? eks + 32 * i : NULL);
}
/* -1, or the lowest parent index an in-range row names whose sk >= r_J (nothing written) */
EXPORT long long hdo_xsk_derive(size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *pidx, const uint32_t *cidx, uint8_t *xsks,
                                uint8_t *xpgks, uint8_t *dks, uint8_t *eks, uint8_t *status) {
    long long bad = -1;
    for (size_t i = 0; i < n; i++)
        if (pidx[i] < n_parents && !fs_lt(parents + XK * (size_t)pidx[i] + 41) && (bad < 0 || pidx[i] < bad)) bad = pidx[i];
    if (bad >= 0) return bad;
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < nn; i++)
        status[i] = (uint8_t)xsk_child(pidx[i] < n_parents ? parents + XK * (size_t)pidx[i] : NULL, cidx[i], xsks + XK * i,
                                       xpgks ? xpgks + XK * i : NULL, dks ? dks + 32 * i : NULL, eks ? eks + 32 * i : NULL);
    return -1;
}
EXPORT void hdo_xpgk_derive(size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *pidx, const uint32_t *cidx, uint8_t *xpgks,
                            uint8_t *dks, uint8_t *eks, uint8_t *status) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < nn; i++)
        status[i] = (uint8_t)xpgk_child(pidx[i] < n_parents ? parents + XK * (size_t)pidx[i] : NULL, cidx[i], xpgks + XK * i,
                                        dks ? dks + 32 * i : NULL, eks ? eks + 32 * i : NULL);
}
