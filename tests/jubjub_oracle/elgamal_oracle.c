/* TEST INFRASTRUCTURE (oracle) — lifted-ElGamal balance decryption with the Diversifier generator, in plain C99 + OpenMP.
 * Not part of the product; the tests and tools/elgamal_bench.py build it through tests/jubjub_oracle/eg_coracle.py.
 *
 * It builds on the RedJubjub oracle (redjubjub_oracle.c, included as it is, which includes jubjub_oracle.c): Fr, Fs,
 * Point::read, the group law, P_G, Point::mul and Point::write.  Added here:
 *   encrypt / neg_encrypt   core/crypto/src/elgamal.rs:49-85
 *   decrypt                 what zface's BalanceQuery runs (zface/src/utils/getter.rs:135-175): DecryptionKey::read,
 *                           Ciphertext::read of the balance and of the pending transfer (Point::read + as_prime_order),
 *                           add, then the reference's own loop (elgamal.rs:87-110): acc = O, compare the whole point,
 *                           acc += P_G, up to 10^6 times, early exit included.  Ciphertexts are split over the OpenMP
 *                           threads; it is the host-core baseline of the device decryption.
 *   multiples               the encodings of i P_G for i < n by plain successive addition from O */
#include "redjubjub_oracle.c"
#include <stdlib.h>

#define EG_BOUND 1000000u

/* Point::read + as_prime_order: 0 ok */
static int read_prime(const uint8_t *enc, ext_t *p) {
    if (read_point(enc, p)) return 1;
    ext_t t;
    ext_mul(&t, p, JJ_ORDER);
    return !(fr_is_zero(&t.x) && fr_eq(&t.y, &t.z));
}

/* status and value of zk_elgamal_decrypt_batch for one ciphertext; pend may be NULL */
static int eg_decrypt(const uint8_t *dkb, const uint8_t *ct, const uint8_t *pend, uint32_t *value) {
    uint64_t dk[4];
    *value = 0;
    load_le(dk, dkb, 4);
    if (fs_raw_geq(dk, JJ_ORDER)) return 2;                        /* DecryptionKey::read: NotInField */
    ext_t l, r, pl, pr, v, g, acc;
    fr_t d2, zi, x, y, u;
    jj_d2(&d2);
    if (read_prime(ct, &l) || read_prime(ct + 32, &r)) return 3;
    if (pend) {
        if (read_prime(pend, &pl) || read_prime(pend + 32, &pr)) return 4;
        ext_add(&l, &l, &pl, &d2);
        ext_add(&r, &r, &pr, &d2);
    }
    ext_mul(&v, &r, dk);
    ext_neg(&v, &v);
    ext_add(&v, &l, &v, &d2);
    fr_inv(&zi, &v.z);
    fr_mul(&x, &v.x, &zi); fr_mul(&y, &v.y, &zi);
    ext_zero(&acc);
    ext_pg(&g);
    for (uint32_t i = 0; i < EG_BOUND; i++) {
        /* acc == V as projective points: X_acc == x Z_acc and Y_acc == y Z_acc */
        fr_mul(&u, &x, &acc.z);
        if (fr_eq(&u, &acc.x)) {
            fr_mul(&u, &y, &acc.z);
            if (fr_eq(&u, &acc.y)) { *value = i; return 0; }
        }
        ext_add(&acc, &acc, &g, &d2);
    }
    return 1;
}

EXPORT void ego_decrypt(size_t n, const uint8_t *dks, const uint8_t *cts, const uint8_t *pending, uint32_t *values, uint8_t *status) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 1)
    for (long long i = 0; i < nn; i++)
        status[i] = (uint8_t)eg_decrypt(dks + 32 * i, cts + 64 * i, pending ? pending + 64 * i : NULL, values + i);
}

/* Ciphertext::encrypt (neg = 0) or neg_encrypt (neg = 1) of amounts[i] with randomness rs[i] (canonical, < r_J) to the
 * encryption key eks[i] (a valid encoding) */
EXPORT void ego_encrypt(size_t n, const uint32_t *amounts, const uint8_t *rs, const uint8_t *eks, int neg, uint8_t *cts) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 4)
    for (long long i = 0; i < nn; i++) {
        uint64_t r[4], a[4] = {amounts[i], 0, 0, 0};
        ext_t g, ek, left, right, rk;
        fr_t d2;
        jj_d2(&d2);
        load_le(r, rs + 32 * i, 4);
        ext_pg(&g);
        read_point(eks + 32 * i, &ek);
        ext_mul(&right, &g, r);
        ext_mul(&left, &g, a);
        if (neg) ext_neg(&left, &left);
        ext_mul(&rk, &ek, r);
        ext_add(&left, &left, &rk, &d2);
        ext_write(cts + 64 * i, &left);
        ext_write(cts + 64 * i + 32, &right);
    }
}

/* out[32 i ..] = Point::write(i P_G) for i < n: acc = O, then acc += P_G, one addition after another (the normalisation of
 * each block is split over the threads) */
EXPORT void ego_multiples(size_t n, uint8_t *out) {
    enum { BLK = 1 << 16 };
    ext_t *buf = (ext_t *)malloc(sizeof(ext_t) * BLK), acc, g;
    fr_t d2;
    jj_d2(&d2);
    ext_zero(&acc);
    ext_pg(&g);
    for (size_t b = 0; b < n; b += BLK) {
        long long m = (long long)(n - b < BLK ? n - b : BLK);
        for (long long j = 0; j < m; j++) { buf[j] = acc; ext_add(&acc, &acc, &g, &d2); }
#pragma omp parallel for schedule(static)
        for (long long j = 0; j < m; j++) ext_write(out + 32 * (b + j), &buf[j]);
    }
    free(buf);
}
