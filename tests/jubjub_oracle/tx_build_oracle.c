/* TEST INFRASTRUCTURE (oracle) — the sender side of a confidential transfer with the Diversifier generator, in plain C99 +
 * OpenMP.  Not part of the product; the tests and tools/tx_build_bench.py build it through tests/jubjub_oracle/tx_coracle.py.
 *
 * It builds on the ElGamal oracle (elgamal_oracle.c, included as it is, which includes redjubjub_oracle.c and
 * jubjub_oracle.c): Fr, Fs, Point::read, the group law, P_G, Point::mul, Point::write, BLAKE2b and signing.  Added here,
 * each step the reference's way, every product its own double-and-add:
 *   BLAKE2s-256              RFC 7693, no key or salt, an 8-byte personalization
 *   keys                     SpendingKey::from_seed, ProofGenerationKey, into_decryption_key, EncryptionKey
 *                            (core/keys/src/lib.rs:64-71, 167-199)
 *   g_epoch                  GEpoch::group_hash: tag bytes from 0, Point::read, mul_by_cofactor, not O; the reference
 *                            asserts after hashing tag 255, so 0..254 are the usable tags (core/primitives/src/g_epoch.rs:102-145)
 *   fields                   MultiCiphertexts::<Confidential>::encrypt (amount P_G + r ek for both keys, fee P_G + r ek_s,
 *                            r P_G), rvk = pgk + alpha P_G, nonce = dk g_epoch, rsk = sk + alpha, in the layout of
 *                            zk_confidential_fields_batch
 * Rows are split over the OpenMP threads; it is the host-core baseline of the device calls. */
#include "elgamal_oracle.c"

/* ---- BLAKE2s-256, written from RFC 7693 ---- */
static const uint32_t B2S_IV[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
typedef struct { uint32_t h[8]; uint8_t buf[64]; size_t fill; uint32_t total; } b2s_t;

static uint32_t le32(const uint8_t *b) { return (uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24); }
static uint32_t rotr32(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
static void b2s_mix(uint32_t *v, int a, int b, int c, int d, uint32_t x, uint32_t y) {
    v[a] += v[b] + x; v[d] = rotr32(v[d] ^ v[a], 16); v[c] += v[d]; v[b] = rotr32(v[b] ^ v[c], 12);
    v[a] += v[b] + y; v[d] = rotr32(v[d] ^ v[a], 8); v[c] += v[d]; v[b] = rotr32(v[b] ^ v[c], 7);
}
static void b2s_block(b2s_t *s, int last) {
    uint32_t m[16], v[16];
    for (int i = 0; i < 16; i++) m[i] = le32(s->buf + 4 * i);
    for (int i = 0; i < 8; i++) { v[i] = s->h[i]; v[i + 8] = B2S_IV[i]; }
    v[12] ^= s->total;
    if (last) v[14] = ~v[14];
    for (int r = 0; r < 10; r++) {
        const uint8_t *z = B2B_SIGMA[r];
        b2s_mix(v, 0, 4, 8, 12, m[z[0]], m[z[1]]);  b2s_mix(v, 1, 5, 9, 13, m[z[2]], m[z[3]]);
        b2s_mix(v, 2, 6, 10, 14, m[z[4]], m[z[5]]); b2s_mix(v, 3, 7, 11, 15, m[z[6]], m[z[7]]);
        b2s_mix(v, 0, 5, 10, 15, m[z[8]], m[z[9]]); b2s_mix(v, 1, 6, 11, 12, m[z[10]], m[z[11]]);
        b2s_mix(v, 2, 7, 8, 13, m[z[12]], m[z[13]]); b2s_mix(v, 3, 4, 9, 14, m[z[14]], m[z[15]]);
    }
    for (int i = 0; i < 8; i++) s->h[i] ^= v[i] ^ v[i + 8];
}
/* 32-byte digest, no key, no salt, 8-byte personalization (parameter block bytes 24..31) */
static void b2s_init(b2s_t *s, const uint8_t *person) {
    for (int i = 0; i < 8; i++) s->h[i] = B2S_IV[i];
    s->h[0] ^= 0x01010020u;
    s->h[6] ^= le32(person); s->h[7] ^= le32(person + 4);
    s->fill = 0; s->total = 0;
}
static void b2s_update(b2s_t *s, const uint8_t *in, size_t len) {
    for (size_t i = 0; i < len; i++) {
        if (s->fill == 64) { s->total += 64; b2s_block(s, 0); s->fill = 0; }
        s->buf[s->fill++] = in[i];
    }
}
static void b2s_final(b2s_t *s, uint8_t *out) {
    s->total += (uint32_t)s->fill;
    memset(s->buf + s->fill, 0, 64 - s->fill);
    b2s_block(s, 1);
    for (int i = 0; i < 32; i++) out[i] = (uint8_t)(s->h[i / 4] >> (8 * (i % 4)));
}

/* ---- keys ---- */
static const uint8_t EXPAND_SEED_PERSONAL[16] = {'z', 'e', 'c', 'h', '_', 'E', 'x', 'p', 'a', 'n', 'd', 'S', 'e', 'e', 'd', '_'};
static const uint8_t BDK_PERSONAL[8] = {'z', 'e', 'c', 'h', '_', 'b', 'd', 'k'};
static const uint8_t GEPOCH_PERSONAL[8] = {'z', 'c', 'g', 'e', 'p', 'o', 'c', 'h'};
static const char GH_FIRST_BLOCK[] = "096b36a5804bfacef1691e173c366a47ff5ba84a44f26ddd7e8d9f79d5b42df0";   /* constants.rs:5-6 */

static void spending_key(uint64_t *sk, const uint8_t *seed, size_t len) {
    b2b_t s;
    uint8_t d[64];
    b2b_init(&s, EXPAND_SEED_PERSONAL);
    b2b_update(&s, seed, len);
    b2b_final(&s, d);
    to_uniform(sk, d);
}
/* ProofGenerationKey (sk P_G) -> into_decryption_key */
static void decryption_key(uint64_t *dk, ext_t *pgk, const uint64_t *sk) {
    ext_t g;
    uint8_t enc[32], h[32];
    b2s_t s;
    ext_pg(&g);
    ext_mul(pgk, &g, sk);
    ext_write(enc, pgk);
    b2s_init(&s, BDK_PERSONAL);
    b2s_update(&s, enc, 32);
    b2s_final(&s, h);
    h[31] &= 0x07;
    load_le(dk, h, 4);
}
static void pg_mul(ext_t *r, const uint64_t *k) { ext_t g; ext_pg(&g); ext_mul(r, &g, k); }
static void store_le(uint8_t *b, const uint64_t *w) { for (int i = 0; i < 32; i++) b[i] = (uint8_t)(w[i / 8] >> (8 * (i % 8))); }

/* ---- GEpoch::group_hash: 1 and the tag byte, or 0 ---- */
static int g_epoch(uint8_t *out, uint32_t epoch, int *tag) {
    for (int i = 0; i < 255; i++) {
        uint8_t e[5] = {(uint8_t)epoch, (uint8_t)(epoch >> 8), (uint8_t)(epoch >> 16), (uint8_t)(epoch >> 24), (uint8_t)i}, h[32];
        b2s_t s;
        b2s_init(&s, GEPOCH_PERSONAL);
        b2s_update(&s, (const uint8_t *)GH_FIRST_BLOCK, 64);
        b2s_update(&s, e, 5);
        b2s_final(&s, h);
        ext_t p;
        if (read_point(h, &p)) continue;
        for (int k = 0; k < 3; k++) ext_dbl(&p, &p);
        if (fr_is_zero(&p.x) && fr_eq(&p.y, &p.z)) continue;
        ext_write(out, &p);
        *tag = i;
        return 1;
    }
    return 0;
}

/* ---- one row of zk_confidential_fields_batch; returns its status ---- */
static int tx_fields(uint8_t *f, uint8_t *rskb, uint8_t *dkb, const uint8_t *skb, const uint8_t *ekb, uint32_t amount, uint32_t fee,
                     const uint8_t *rb, const uint8_t *alb, const ext_t *g, const uint8_t *g_enc) {
    ext_t ekr, t;
    int st = read_point(ekb, &ekr);
    if (!st) {
        ext_mul(&t, &ekr, JJ_ORDER);
        if (!(fr_is_zero(&t.x) && fr_eq(&t.y, &t.z))) st = 3;
    }
    if (st) {
        memset(f, 0, 288); memset(rskb, 0, 32); memset(dkb, 0, 32);
        return st;
    }
    uint64_t sk[4], r[4], al[4], dk[4], am[4] = {amount, 0, 0, 0}, fe[4] = {fee, 0, 0, 0}, rsk[4];
    load_le(sk, skb, 4); load_le(r, rb, 4); load_le(al, alb, 4);
    ext_t pgk, eks, a, b, c, rpg, rvk, nonce;
    fr_t d2;
    jj_d2(&d2);
    decryption_key(dk, &pgk, sk);
    pg_mul(&eks, dk);
    ext_write(f, &eks);                                              /* address_sender */
    memcpy(f + 32, ekb, 32);                                         /* address_recipient */
    pg_mul(&rpg, r);
    pg_mul(&a, am); ext_mul(&b, &eks, r); ext_add(&c, &a, &b, &d2); ext_write(f + 64, &c);    /* amount_sender */
    ext_mul(&b, &ekr, r); ext_add(&c, &a, &b, &d2); ext_write(f + 96, &c);                   /* amount_recipient */
    pg_mul(&a, fe); ext_mul(&b, &eks, r); ext_add(&c, &a, &b, &d2); ext_write(f + 128, &c);  /* fee_sender */
    ext_write(f + 160, &rpg);                                        /* randomness */
    pg_mul(&a, al); ext_add(&rvk, &pgk, &a, &d2); ext_write(f + 192, &rvk);
    memcpy(f + 224, g_enc, 32);                                      /* g_epoch */
    ext_mul(&nonce, g, dk); ext_write(f + 256, &nonce);
    fs_t fsk, fal;
    fs_from_repr(&fsk, sk); fs_from_repr(&fal, al);
    fs_add(&fsk, &fsk, &fal);
    fs_into_repr(rsk, &fsk);
    store_le(rskb, rsk);
    store_le(dkb, dk);
    return 0;
}

EXPORT void txo_blake2s(const uint8_t *person, const uint8_t *in, size_t len, uint8_t *out) {
    b2s_t s;
    b2s_init(&s, person);
    b2s_update(&s, in, len);
    b2s_final(&s, out);
}
EXPORT void txo_keys(size_t n, const uint8_t *seeds, const uint64_t *off, uint8_t *sks, uint8_t *dks, uint8_t *eks) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < nn; i++) {
        uint64_t sk[4], dk[4];
        ext_t pgk, ek;
        spending_key(sk, seeds + off[i], off[i + 1] - off[i]);
        decryption_key(dk, &pgk, sk);
        pg_mul(&ek, dk);
        store_le(sks + 32 * i, sk); store_le(dks + 32 * i, dk); ext_write(eks + 32 * i, &ek);
    }
}
/* tags[i]: the tag byte GEpoch::group_hash(epochs[i]) took, or -1 (out[i] then unset) */
EXPORT void txo_g_epoch(size_t n, const uint32_t *epochs, uint8_t *out, int32_t *tags) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 1)
    for (long long i = 0; i < nn; i++) {
        int tag = -1;
        if (!g_epoch(out + 32 * i, epochs[i], &tag)) tag = -1;
        tags[i] = tag;
    }
}
/* 0, or 1 when g_epoch fails Point::read + as_prime_order (nothing written); scalars canonical */
EXPORT int txo_fields(size_t n, const uint8_t *sks, const uint8_t *eks, const uint32_t *amounts, const uint32_t *fees, const uint8_t *rs,
                      const uint8_t *alphas, const uint8_t *g_enc, uint8_t *fields, uint8_t *rsks, uint8_t *dks, uint8_t *status) {
    ext_t g;
    if (read_prime(g_enc, &g)) return 1;
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 4)
    for (long long i = 0; i < nn; i++)
        status[i] = (uint8_t)tx_fields(fields + 288 * i, rsks + 32 * i, dks + 32 * i, sks + 32 * i, eks + 32 * i, amounts[i], fees[i],
                                       rs + 32 * i, alphas + 32 * i, &g, g_enc);
    return 0;
}
