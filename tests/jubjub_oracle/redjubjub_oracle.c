/* TEST INFRASTRUCTURE (oracle) — RedJubjub verification with the Diversifier generator, in plain C99 + OpenMP.  Not part of
 * the product; the tests and tools/redjubjub_bench.py build it through tests/jubjub_oracle/rj_coracle.py.
 *
 * It builds on the Jubjub point decoder's oracle (jubjub_oracle.c, included as it is): its Fr arithmetic on
 * oracle/field_tmpl.inc, the Tonelli-Shanks square root and the extended-coordinate group law.  Added here: Point::read without
 * the subgroup test, BLAKE2b, Fs, and the signature itself.  Several signatures are split over the OpenMP threads; it is the
 * host-core baseline of the device verifier. */
#include "jubjub_oracle.c"

static void load_le(uint64_t *w, const uint8_t *b, int nw) {
    for (int i = 0; i < nw; i++) { w[i] = 0; for (int k = 0; k < 8; k++) w[i] |= (uint64_t)b[8 * i + k] << (8 * k); }
}

/* Point::read (core/jubjub/src/curve/edwards.rs:92-164), Unknown order: 0 ok (p = (x, y, 1, xy)), 1 NotInField, 2 NotOnCurve */
static int read_point(const uint8_t *enc, ext_t *p) {
    uint64_t yr[4], xr[4];
    load_le(yr, enc, 4);
    int sign = (int)(yr[3] >> 63);
    yr[3] &= 0x7fffffffffffffffULL;
    fr_t y, one, d, y2, num, den, x;
    if (fr_from_repr(&y, yr)) return 1;
    fr_set_one(&one);
    fr_const(&d, JJ_D);
    fr_sqr(&y2, &y);
    fr_mul(&den, &y2, &d); fr_add(&den, &den, &one);
    fr_sub(&num, &y2, &one);
    if (fr_inv(&den, &den)) return 2;                      /* cannot happen: d is not a square */
    fr_mul(&num, &num, &den);
    if (fr_sqrt(&x, &num)) return 2;
    fr_into_repr(xr, &x);
    if ((int)(xr[0] & 1) != sign) fr_neg(&x, &x);
    p->x = x; p->y = y; fr_set_one(&p->z); fr_mul(&p->t, &x, &y);
    return 0;
}

static void jj_d2(fr_t *d2) { fr_const(d2, JJ_D); fr_dbl(d2, d2); }
/* ==== RedJubjub with the Diversifier generator (core/jubjub/src/redjubjub.rs) ============================================
 *   H*(a || b)   BLAKE2b-512 (RFC 7693), personalization "Zcash_RedJubjubH", then Fs::to_uniform the reference's way:
 *                one.mul_bits over the 512 digest bits, most significant first (curve/fs.rs:587-592)
 *   sign         redjubjub.rs:73-103 with T supplied by the caller
 *   verify       redjubjub.rs:127-155: c vk + R + -(S P_G), mul_by_cofactor, == O; each product its own double-and-add */

/* ---- BLAKE2b, written from RFC 7693 ---- */
static const uint64_t B2B_IV[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                   0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
static const uint8_t B2B_SIGMA[12][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};

typedef struct { uint64_t h[8]; uint8_t buf[128]; size_t fill; uint64_t total; } b2b_t;

static uint64_t rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
static void b2b_mix(uint64_t *v, int a, int b, int c, int d, uint64_t x, uint64_t y) {
    v[a] += v[b] + x; v[d] = rotr(v[d] ^ v[a], 32); v[c] += v[d]; v[b] = rotr(v[b] ^ v[c], 24);
    v[a] += v[b] + y; v[d] = rotr(v[d] ^ v[a], 16); v[c] += v[d]; v[b] = rotr(v[b] ^ v[c], 63);
}
static void b2b_block(b2b_t *s, int last) {
    uint64_t m[16], v[16];
    load_le(m, s->buf, 16);
    for (int i = 0; i < 8; i++) { v[i] = s->h[i]; v[i + 8] = B2B_IV[i]; }
    v[12] ^= s->total;
    if (last) v[14] = ~v[14];
    for (int r = 0; r < 12; r++) {
        const uint8_t *z = B2B_SIGMA[r];
        b2b_mix(v, 0, 4, 8, 12, m[z[0]], m[z[1]]);  b2b_mix(v, 1, 5, 9, 13, m[z[2]], m[z[3]]);
        b2b_mix(v, 2, 6, 10, 14, m[z[4]], m[z[5]]); b2b_mix(v, 3, 7, 11, 15, m[z[6]], m[z[7]]);
        b2b_mix(v, 0, 5, 10, 15, m[z[8]], m[z[9]]); b2b_mix(v, 1, 6, 11, 12, m[z[10]], m[z[11]]);
        b2b_mix(v, 2, 7, 8, 13, m[z[12]], m[z[13]]); b2b_mix(v, 3, 4, 9, 14, m[z[14]], m[z[15]]);
    }
    for (int i = 0; i < 8; i++) s->h[i] ^= v[i] ^ v[i + 8];
}
/* 64-byte digest, no key, no salt, 16-byte personalization (parameter block bytes 48..63) */
static void b2b_init(b2b_t *s, const uint8_t *person) {
    uint64_t p[2];
    load_le(p, person, 2);
    for (int i = 0; i < 8; i++) s->h[i] = B2B_IV[i];
    s->h[0] ^= 0x01010040ULL;
    s->h[6] ^= p[0]; s->h[7] ^= p[1];
    s->fill = 0; s->total = 0;
}
static void b2b_update(b2b_t *s, const uint8_t *in, size_t len) {
    for (size_t i = 0; i < len; i++) {
        if (s->fill == 128) { s->total += 128; b2b_block(s, 0); s->fill = 0; }   /* a full buffer is compressed only once more input comes */
        s->buf[s->fill++] = in[i];
    }
}
static void b2b_final(b2b_t *s, uint8_t *out) {
    s->total += s->fill;
    memset(s->buf + s->fill, 0, 128 - s->fill);
    b2b_block(s, 1);
    for (int i = 0; i < 64; i++) out[i] = (uint8_t)(s->h[i / 8] >> (8 * (i % 8)));
}

/* ---- Fs (fs.rs): r_J, R = 2^256 ---- */
#undef FN
#undef FT
#undef F_MODULUS
#undef F_R
#undef F_R2
#undef F_INV
typedef struct { uint64_t l[4]; } fs_t;
static const uint64_t FS_R[4] = {0x25f80bb3b99607d9ULL, 0xf315d62f66b6e750ULL, 0x932514eeeb8814f4ULL, 0x09a6fc6f479155c6ULL};
static const uint64_t FS_R2[4] = {0x67719aa495e57731ULL, 0x51b0cef09ce3fc26ULL, 0x69dab7fac026e9a5ULL, 0x04f6547b8d127688ULL};
#define FN(x) CAT(fs_, x)
#define FT fs_t
#define F_MODULUS JJ_ORDER
#define F_R FS_R
#define F_R2 FS_R2
#define F_INV 0x1ba3a358ef788ef9ULL
#include "field_tmpl.inc"

static const uint8_t H_STAR_PERSONAL[16] = {'Z', 'c', 'a', 's', 'h', '_', 'R', 'e', 'd', 'J', 'u', 'b', 'j', 'u', 'b', 'H'};

/* Fs::to_uniform: one.mul_bits(BitIterator(digest as 8 LE u64)), returned canonical */
static void to_uniform(uint64_t *out, const uint8_t *digest) {
    uint64_t w[8];
    load_le(w, digest, 8);
    fs_t acc, one;
    fs_set_zero(&acc); fs_set_one(&one);
    for (int i = 511; i >= 0; i--) {
        fs_dbl(&acc, &acc);
        if ((w[i / 64] >> (i % 64)) & 1) fs_add(&acc, &acc, &one);
    }
    fs_into_repr(out, &acc);
}
static void h_star(uint64_t *out, const uint8_t *a, size_t alen, const uint8_t *b, size_t blen) {
    b2b_t s;
    uint8_t d[64];
    b2b_init(&s, H_STAR_PERSONAL);
    b2b_update(&s, a, alen);
    b2b_update(&s, b, blen);
    b2b_final(&s, d);
    to_uniform(out, d);
}

/* ---- Jubjub points ---- */
/* P_G = find_group_hash(b"r", "Zcash_PH") (curve/mod.rs:325-326), canonical; the tests pin it to the Python oracle's */
static const uint64_t PG_X[4] = {0xa5143b34a8e36462ULL, 0xf0919d06ffb1ecdaULL, 0xa1409aa1f33bec2cULL, 0x26eb9f8a9ec72a8cULL};
static const uint64_t PG_Y[4] = {0xd4fc6365796c77acULL, 0x96b78beafa9cc44cULL, 0x949d77476e262c95ULL, 0x114b7501ad104c57ULL};

static void ext_zero(ext_t *p) { fr_set_zero(&p->x); fr_set_one(&p->y); fr_set_one(&p->z); fr_set_zero(&p->t); }
static void ext_pg(ext_t *p) {
    fr_const(&p->x, PG_X); fr_const(&p->y, PG_Y); fr_set_one(&p->z); fr_mul(&p->t, &p->x, &p->y);
}
static void ext_neg(ext_t *r, const ext_t *p) { *r = *p; fr_neg(&r->x, &p->x); fr_neg(&r->t, &p->t); }
/* Point::mul: double-and-add over the 256 bits of a canonical scalar */
static void ext_mul(ext_t *r, const ext_t *p, const uint64_t *k) {
    fr_t d2; jj_d2(&d2);
    ext_t acc; ext_zero(&acc);
    for (int i = 255; i >= 0; i--) {
        ext_dbl(&acc, &acc);
        if ((k[i / 64] >> (i % 64)) & 1) ext_add(&acc, &acc, p, &d2);
    }
    *r = acc;
}
/* Point::write: y with the parity of x in bit 255 */
static void ext_write(uint8_t *out, const ext_t *p) {
    fr_t zi, x, y;
    uint64_t xr[4], yr[4];
    fr_inv(&zi, &p->z);
    fr_mul(&x, &p->x, &zi); fr_mul(&y, &p->y, &zi);
    fr_into_repr(xr, &x); fr_into_repr(yr, &y);
    yr[3] |= (xr[0] & 1) << 63;
    for (int i = 0; i < 32; i++) out[i] = (uint8_t)(yr[i / 8] >> (8 * (i % 8)));
}

/* verdicts of zk_redjubjub_verify_batch: 1 true, 0 equation fails, 2 bad vk, 3 bad rbar, 4 sbar >= r_J */
static int rj_verify(const uint8_t *vk, const uint8_t *sig, const uint8_t *msg, size_t mlen) {
    uint64_t c[4], s[4];
    h_star(c, sig, 32, msg, mlen);
    ext_t a, r, t, u;
    if (read_point(vk, &a)) return 2;
    if (read_point(sig, &r)) return 3;
    load_le(s, sig + 32, 4);
    if (fs_raw_geq(s, JJ_ORDER)) return 4;
    fr_t d2; jj_d2(&d2);
    ext_mul(&t, &a, c);
    ext_add(&t, &t, &r, &d2);
    ext_pg(&u);
    ext_mul(&u, &u, s);
    ext_neg(&u, &u);
    ext_add(&t, &t, &u, &d2);
    for (int i = 0; i < 3; i++) ext_dbl(&t, &t);
    return fr_is_zero(&t.x) && fr_eq(&t.y, &t.z);
}
/* PrivateKey::sign with T = t (80 bytes); sk canonical < r_J */
static void rj_sign(uint8_t *sig, const uint8_t *skb, const uint8_t *t, const uint8_t *msg, size_t mlen) {
    uint64_t r[4], c[4], skr[4], sr[4];
    h_star(r, t, 80, msg, mlen);
    ext_t g, rg;
    ext_pg(&g);
    ext_mul(&rg, &g, r);
    ext_write(sig, &rg);
    h_star(c, sig, 32, msg, mlen);
    load_le(skr, skb, 4);
    fs_t fc, fsk, fr_;
    fs_from_repr(&fc, c); fs_from_repr(&fsk, skr); fs_from_repr(&fr_, r);
    fs_mul(&fc, &fc, &fsk);
    fs_add(&fc, &fc, &fr_);
    fs_into_repr(sr, &fc);
    for (int i = 0; i < 32; i++) sig[32 + i] = (uint8_t)(sr[i / 8] >> (8 * (i % 8)));
}

EXPORT void rjo_verify(size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *off, uint8_t *verdicts) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < nn; i++)
        verdicts[i] = (uint8_t)rj_verify(vks + 32 * i, sigs + 64 * i, msgs + off[i], off[i + 1] - off[i]);
}
EXPORT void rjo_sign(size_t n, const uint8_t *sks, const uint8_t *ts, const uint8_t *msgs, const uint64_t *off, uint8_t *sigs) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < nn; i++) rj_sign(sigs + 64 * i, sks + 32 * i, ts + 80 * i, msgs + off[i], off[i + 1] - off[i]);
}
/* PublicKey::from_private: sk P_G, encoded */
EXPORT void rjo_public_key(size_t n, const uint8_t *sks, uint8_t *vks) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < nn; i++) {
        uint64_t k[4];
        ext_t g, p;
        load_le(k, sks + 32 * i, 4);
        ext_pg(&g);
        ext_mul(&p, &g, k);
        ext_write(vks + 32 * i, &p);
    }
}
/* H*(a || b), canonical */
EXPORT void rjo_h_star(const uint8_t *a, size_t alen, const uint8_t *b, size_t blen, uint64_t *out) { h_star(out, a, alen, b, blen); }
/* plain BLAKE2b-512 with a 16-byte personalization (for the RFC 7693 check, person = 16 zero bytes) */
EXPORT void rjo_blake2b(const uint8_t *person, const uint8_t *in, size_t len, uint8_t *out) {
    b2b_t s;
    b2b_init(&s, person);
    b2b_update(&s, in, len);
    b2b_final(&s, out);
}
