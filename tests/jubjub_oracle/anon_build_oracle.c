/* TEST INFRASTRUCTURE (oracle) — the sender side of an anonymous transfer with the Diversifier generator, in plain C99 +
 * OpenMP.  Not part of the product; the tests and tools/anon_build_bench.py build it through
 * tests/jubjub_oracle/anon_build_coracle.py.
 *
 * It builds on the transaction-building oracle (tx_build_oracle.c, included as it is, which includes elgamal_oracle.c,
 * redjubjub_oracle.c and jubjub_oracle.c): key derivation, P_G, Point::read, Point::mul, Point::write.  Added here, each
 * step the reference's way, every product its own double-and-add:
 *   anonymous fields         MultiCiphertexts::<Anonymous>::encrypt (neg_encrypt for the sender, encrypt for the
 *                            recipient, encrypt(0) for each decoy; core/proofs/src/crypto_components.rs:168-216), placed by
 *                            replaying gen_proof's two Vec::insert calls (core/proofs/src/anonymous.rs:118-145), with rvk,
 *                            nonce, rsk and dk, in the layout of zk_anonymous_fields_batch
 * Rows are split over the OpenMP threads; it is the host-core baseline of the device call. */
#include "tx_build_oracle.c"

/* ---- one row of zk_anonymous_fields_batch; returns its status ---- */
/* Vec::insert(at, x) on a vector of len 32-byte items */
static void vec_insert(uint8_t *v, int len, int at, const uint8_t *x) {
    memmove(v + 32 * (at + 1), v + 32 * at, 32 * (size_t)(len - at));
    memcpy(v + 32 * at, x, 32);
}
/* MultiCiphertexts' ciphertext of amount under ek: -amount P_G + r ek for neg, amount P_G + r ek otherwise (amount 0 for
 * a decoy); each product its own double-and-add */
static void eg_left(uint8_t *out, uint32_t amount, int neg, const uint64_t *r, const ext_t *ek) {
    uint64_t a[4] = {amount, 0, 0, 0};
    ext_t left, rk;
    fr_t d2;
    jj_d2(&d2);
    pg_mul(&left, a);
    if (neg) ext_neg(&left, &left);
    ext_mul(&rk, ek, r);
    ext_add(&left, &left, &rk, &d2);
    ext_write(out, &left);
}
static int anon_fields(uint8_t *f, uint8_t *rskb, uint8_t *dkb, size_t n_keys, const uint8_t *keys, const uint32_t *ring, int s, int t,
                       const uint8_t *skb, uint32_t amount, const uint8_t *rb, const uint8_t *alb, const ext_t *g) {
    ext_t ek[11];
    int st = 0;
    if (s >= 12 || t >= 12 || s == t) st = 5;
    for (int j = 0; j < 11 && !st; j++)
        if (ring[j] >= n_keys) st = 4;
    for (int j = 0; j < 11 && !st; j++) {
        st = read_point(keys + 32 * (size_t)ring[j], &ek[j]);
        if (!st) {
            ext_t o;
            ext_mul(&o, &ek[j], JJ_ORDER);
            if (!(fr_is_zero(&o.x) && fr_eq(&o.y, &o.z))) st = 3;
        }
    }
    if (st) {
        memset(f, 0, 864); memset(rskb, 0, 32); memset(dkb, 0, 32);
        return st;
    }
    uint64_t sk[4], r[4], al[4], dk[4], rsk[4];
    load_le(sk, skb, 4); load_le(r, rb, 4); load_le(al, alb, 4);
    ext_t pgk, eks, a, rvk, right, nonce;
    fr_t d2;
    jj_d2(&d2);
    decryption_key(dk, &pgk, sk);
    pg_mul(&eks, dk);
    uint8_t keys_v[12 * 32], lefts_v[12 * 32], ek_s[32], left_s[32], left_t[32];
    for (int j = 1; j < 11; j++) {                               /* the decoys in order */
        memcpy(keys_v + 32 * (j - 1), keys + 32 * (size_t)ring[j], 32);
        eg_left(lefts_v + 32 * (j - 1), 0, 0, r, &ek[j]);
    }
    ext_write(ek_s, &eks);
    eg_left(left_s, amount, 1, r, &eks);                          /* neg_encrypt */
    eg_left(left_t, amount, 0, r, &ek[0]);                        /* encrypt */
    if (s < t) {
        vec_insert(keys_v, 10, s, ek_s); vec_insert(keys_v, 11, t, keys + 32 * (size_t)ring[0]);
        vec_insert(lefts_v, 10, s, left_s); vec_insert(lefts_v, 11, t, left_t);
    } else {
        vec_insert(keys_v, 10, t, keys + 32 * (size_t)ring[0]); vec_insert(keys_v, 11, s, ek_s);
        vec_insert(lefts_v, 10, t, left_t); vec_insert(lefts_v, 11, s, left_s);
    }
    memcpy(f, keys_v, 384);
    memcpy(f + 384, lefts_v, 384);
    pg_mul(&right, r); ext_write(f + 768, &right);                /* right_ciphertext */
    pg_mul(&a, al); ext_add(&rvk, &pgk, &a, &d2); ext_write(f + 800, &rvk);
    ext_mul(&nonce, g, dk); ext_write(f + 832, &nonce);
    fs_t fsk, fal;
    fs_from_repr(&fsk, sk); fs_from_repr(&fal, al);
    fs_add(&fsk, &fsk, &fal);
    fs_into_repr(rsk, &fsk);
    store_le(rskb, rsk);
    store_le(dkb, dk);
    return 0;
}

/* 0, or 1 when g_epoch fails Point::read + as_prime_order (nothing written); scalars canonical.  rings: n * 11 indices,
 * positions: n * 2 bytes */
EXPORT int abo_fields(size_t n_keys, const uint8_t *keys, size_t n, const uint8_t *sks, const uint32_t *rings, const uint8_t *positions,
                      const uint32_t *amounts, const uint8_t *rs, const uint8_t *alphas, const uint8_t *g_enc, uint8_t *fields,
                      uint8_t *rsks, uint8_t *dks, uint8_t *status) {
    ext_t g;
    if (read_prime(g_enc, &g)) return 1;
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 1)
    for (long long i = 0; i < nn; i++)
        status[i] = (uint8_t)anon_fields(fields + 864 * i, rsks + 32 * i, dks + 32 * i, n_keys, keys, rings + 11 * i, positions[2 * i],
                                         positions[2 * i + 1], sks + 32 * i, amounts[i], rs + 32 * i, alphas + 32 * i, &g);
    return 0;
}
