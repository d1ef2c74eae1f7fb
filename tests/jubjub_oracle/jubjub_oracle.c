/* TEST INFRASTRUCTURE (oracle) — Jubjub point decoding in plain C99 + OpenMP on the oracle's Fr arithmetic
 * (oracle/field_tmpl.inc, 64-bit limbs).  Not part of the product; the tests and tools/verify_tx_bench.py build it.
 *
 * Restates, per 32-byte encoding, what modules/zk-system's PublicInputBuilder::push does (input_builder.rs:15-27):
 *   Point::read      core/jubjub/src/curve/edwards.rs:92-164   (y < r, x = sqrt((y^2 - 1) / (d y^2 + 1)), sign fix)
 *   as_prime_order   edwards.rs:319-325                        ([r_J] P == O, projective comparison)
 *   into_xy          edwards.rs:341-352
 * with the reference's own algorithms: Tonelli-Shanks after a Legendre test (fr.rs sqrt), extended coordinates, and a
 * double-and-add over the bits of r_J.  One call decodes n encodings, points split over the OpenMP threads; it is the
 * host-core baseline of the device decoder. */
#include <stdint.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define EXPORT __attribute__((visibility("default")))
#define CAT_(a, b) a##b
#define CAT(a, b) CAT_(a, b)

typedef struct { uint64_t l[4]; } fr_t;
/* fr.rs:4-55 */
static const uint64_t FR_MODULUS[4] = {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL};
static const uint64_t FR_R[4] = {0x00000001fffffffeULL, 0x5884b7fa00034802ULL, 0x998c4fefecbc4ff5ULL, 0x1824b159acc5056fULL};
static const uint64_t FR_R2[4] = {0xc999e990f3f29c6dULL, 0x2b6cedcb87925c23ULL, 0x05d314967254398fULL, 0x0748d9d99f59ff11ULL};
#define FR_INV 0xfffffffeffffffffULL
#define FN(x) CAT(fr_, x)
#define FT fr_t
#define NL 4
#define F_MODULUS FR_MODULUS
#define F_R FR_R
#define F_R2 FR_R2
#define F_INV FR_INV
#include "field_tmpl.inc"

/* canonical constants */
static const uint64_t JJ_D[4] = {0x01065fd6d6343eb1ULL, 0x292d7f6d37579d26ULL, 0xf5fd9207e6bd7fd4ULL, 0x2a9318e74bfa2b48ULL};   /* mod.rs:204 */
static const uint64_t JJ_ORDER[4] = {0xd0970e5ed6f72cb7ULL, 0xa6682093ccc81082ULL, 0x06673b0101343b00ULL, 0x0e7db4ea6533afa9ULL}; /* fs.rs:14 */
#define FR_S 32
static const uint64_t FR_T[4] = {0xfffe5bfeffffffffULL, 0x09a1d80553bda402ULL, 0x299d7d483339d808ULL, 0x0000000073eda753ULL};   /* (r-1)/2^32 */
static const uint64_t FR_T_PLUS1_HALF[4] = {0x7fff2dff80000000ULL, 0x04d0ec02a9ded201ULL, 0x94cebea4199cec04ULL, 0x0000000039f6d3a9ULL};
static const uint64_t FR_HALF_PM1[4] = {0x7fffffff80000000ULL, 0xa9ded2017fff2dffULL, 0x199cec0404d0ec02ULL, 0x39f6d3a994cebea4ULL}; /* (r-1)/2 */
static const uint64_t FR_GEN_CAN[4] = {7, 0, 0, 0};

static void fr_const(fr_t *r, const uint64_t *canonical) { fr_from_repr(r, canonical); }

/* Tonelli-Shanks (r = 2^32 t + 1) after Euler's criterion; returns -1 for a non-residue */
static int fr_sqrt(fr_t *r, const fr_t *a) {
    if (fr_is_zero(a)) { *r = *a; return 0; }
    fr_t one, leg, c, x, b, t2, e;
    fr_set_one(&one);
    fr_pow(&leg, a, FR_HALF_PM1, 4);
    if (!fr_eq(&leg, &one)) return -1;
    fr_const(&c, FR_GEN_CAN);
    fr_pow(&c, &c, FR_T, 4);                 /* 7^t: order 2^32 */
    fr_pow(&x, a, FR_T_PLUS1_HALF, 4);
    fr_pow(&b, a, FR_T, 4);
    int m = FR_S;
    while (!fr_eq(&b, &one)) {
        int i = 0;
        t2 = b;
        while (!fr_eq(&t2, &one)) { fr_sqr(&t2, &t2); i++; }
        e = c;
        for (int j = 0; j < m - i - 1; j++) fr_sqr(&e, &e);
        fr_sqr(&c, &e);
        fr_mul(&x, &x, &e);
        fr_mul(&b, &b, &c);
        m = i;
    }
    *r = x;
    return 0;
}

typedef struct { fr_t x, y, z, t; } ext_t;

static void ext_add(ext_t *r, const ext_t *p, const ext_t *q, const fr_t *d2) {   /* a = -1, k = 2d */
    fr_t a, b, c, d, e, f, g, h, u, v;
    fr_sub(&u, &p->y, &p->x); fr_sub(&v, &q->y, &q->x); fr_mul(&a, &u, &v);
    fr_add(&u, &p->y, &p->x); fr_add(&v, &q->y, &q->x); fr_mul(&b, &u, &v);
    fr_mul(&c, &p->t, d2); fr_mul(&c, &c, &q->t);
    fr_mul(&d, &p->z, &q->z); fr_dbl(&d, &d);
    fr_sub(&e, &b, &a); fr_sub(&f, &d, &c); fr_add(&g, &d, &c); fr_add(&h, &b, &a);
    fr_mul(&r->x, &e, &f); fr_mul(&r->y, &g, &h); fr_mul(&r->t, &e, &h); fr_mul(&r->z, &f, &g);
}
static void ext_dbl(ext_t *r, const ext_t *p) {
    fr_t a, b, c, d, e, f, g, h;
    fr_sqr(&a, &p->x); fr_sqr(&b, &p->y); fr_sqr(&c, &p->z); fr_dbl(&c, &c);
    fr_neg(&d, &a);
    fr_add(&e, &p->x, &p->y); fr_sqr(&e, &e); fr_sub(&e, &e, &a); fr_sub(&e, &e, &b);
    fr_add(&g, &d, &b); fr_sub(&f, &g, &c); fr_sub(&h, &d, &b);
    fr_mul(&r->x, &e, &f); fr_mul(&r->y, &g, &h); fr_mul(&r->t, &e, &h); fr_mul(&r->z, &f, &g);
}

/* status: 0 ok, 1 NotInField, 2 NotOnCurve, 3 not of prime order; xy = canonical x, y (zero when rejected) */
static int into_xy(const uint8_t *enc, uint64_t *xy) {
    uint64_t yr[4];
    memset(xy, 0, 64);
    for (int i = 0; i < 4; i++) { yr[i] = 0; for (int k = 0; k < 8; k++) yr[i] |= (uint64_t)enc[8 * i + k] << (8 * k); }
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
    uint64_t xr[4];
    fr_into_repr(xr, &x);
    if ((int)(xr[0] & 1) != sign) { fr_neg(&x, &x); fr_into_repr(xr, &x); }
    ext_t p, acc;
    p.x = x; p.y = y; fr_set_one(&p.z); fr_mul(&p.t, &x, &y);
    fr_t d2; fr_dbl(&d2, &d);
    acc = p;
    for (int i = 250; i >= 0; i--) {                       /* r_J has 252 bits; bit 251 is the starting value */
        ext_dbl(&acc, &acc);
        if ((JJ_ORDER[i / 64] >> (i % 64)) & 1) ext_add(&acc, &acc, &p, &d2);
    }
    /* == Point::zero(): x1 z2 == x2 z1 and y1 z2 == y2 z1 with (0, 1, 0, 1) */
    if (!fr_is_zero(&acc.x) || !fr_eq(&acc.y, &acc.z)) return 3;
    memcpy(xy, xr, 32);
    fr_into_repr(xy + 4, &y);
    return 0;
}

EXPORT void jjo_into_xy(const uint8_t *enc, size_t n, uint64_t *xy, uint8_t *status) {
    long long nn = (long long)n;
#pragma omp parallel for schedule(dynamic, 64)
    for (long long i = 0; i < nn; i++) status[i] = (uint8_t)into_xy(enc + 32 * i, xy + 8 * i);
}

EXPORT int jjo_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* a square root or -1 (for the square-root tests): in / out canonical */
EXPORT int jjo_sqrt(const uint64_t *a, uint64_t *out) {
    fr_t x, r;
    if (fr_from_repr(&x, a)) return -2;
    if (fr_sqrt(&r, &x)) return -1;
    fr_into_repr(out, &r);
    return 0;
}
