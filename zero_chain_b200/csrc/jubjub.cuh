// Jubjub point decoding over BLS12-381's Fr: the zk-system public-input step (SURVEY.md §8 f2).
//
// Restates, value for value, what modules/zk-system does per public-input point (input_builder.rs:15-27 -> IntoXY):
//   edwards::Point::read      core/jubjub/src/curve/edwards.rs:92-164  y from the low 255 bits (y < r, else NotInField),
//                             x^2 = (y^2 - 1) / (d y^2 + 1), x = sqrt (none: NotOnCurve), x negated when its parity differs
//                             from bit 255
//   as_prime_order            edwards.rs:319-325   [r_J] P == O, else None
//   into_xy                   edwards.rs:341-352   affine (x, y), canonical
// The curve is the twisted Edwards curve -x^2 + y^2 = 1 + d x^2 y^2 (core/jubjub/src/curve/mod.rs:198-210); r_J is the Fs
// modulus (core/jubjub/src/curve/fs.rs:14), the cofactor 8.  Points are kept in extended coordinates (X : Y : Z : T), T = XY/Z,
// with the a = -1 formulas of Hisil-Wong-Carter-Dawson (2008): d is not a square in Fr, so both are complete — no
// exceptional inputs, no branches on point values.
//
// Everything is inlined into the kernel (jubjub.cu): one thread carries a point (32 registers) and a handful of Fr
// temporaries, so there is no call boundary and no stack frame.  The same source compiles with ZK_HOST_EMUL for the CPU test
// (tests/host_emul/emul_jubjub.cpp).
#pragma once
#include "field.cuh"

namespace zkjj {

enum Status : uint8_t { JJ_OK = 0, JJ_NOT_IN_FIELD = 1, JJ_NOT_ON_CURVE = 2, JJ_NOT_PRIME_ORDER = 3 };

// tables walked with a run-time index live in the constant bank (a thread-local array would go to local memory)
#ifdef ZK_HOST_EMUL
#define ZK_JJ_TABLE static const
#else
#define ZK_JJ_TABLE static __device__ __constant__
#endif
// (t - 1) / 2 with r - 1 = 2^32 t, t odd: the exponent of the Tonelli-Shanks start value (222 bits)
ZK_JJ_TABLE uint32_t JJ_SQRT_EXP[7] = {0x7fffffffu, 0x7fff2dffu, 0xa9ded201u, 0x04d0ec02u, 0x199cec04u, 0x94cebea4u, 0x39f6d3a9u};
// r_J = 0x0e7db4ea6533afa906673b0101343b00a6682093ccc81082d0970e5ed6f72cb7 (fs.rs:14), 252 bits
ZK_JJ_TABLE uint32_t JJ_ORDER[8] = {0xd6f72cb7u, 0xd0970e5eu, 0xccc81082u, 0xa6682093u, 0x01343b00u, 0x06673b01u, 0x6533afa9u, 0x0e7db4eau};
constexpr int JJ_ORDER_BITS = 252;
constexpr int FR_TWO_ADICITY = 32;   // fr.rs:47

// canonical constants, turned into Montgomery form where they are used (one product each)
ZK_DEV Fr jj_d2() {    // 2d, d = 19257038036680949359750312669786877991949435402254120286184196891950884077233 (mod.rs:204)
    constexpr uint32_t c[8] = {0xac687d62u, 0x020cbfadu, 0x6eaf3a4cu, 0x525afedau, 0xcd7affa8u, 0xebfb240fu, 0x97f45691u, 0x552631ceu};
    Fr r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.l[i] = c[i];
    return Fr::from_canonical(r);
}
ZK_DEV Fr fr_root_of_unity() {   // 7^t, a generator of the 2^32-torsion of Fr^* (fr.rs:50-55)
    constexpr uint32_t c[8] = {0x439f0d2bu, 0x3829971fu, 0x8c2280b9u, 0xb6368350u, 0x22c813b4u, 0xd09b6819u, 0xdfe81f20u, 0x16a2a19eu};
    Fr r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.l[i] = c[i];
    return Fr::from_canonical(r);
}

// Square root in Fr by Tonelli-Shanks (r = 2^32 t + 1).  Returns false exactly when a is a non-residue; 0 is a square.
// Which of the two roots comes out does not matter: the caller fixes the sign.
ZK_DEV bool fr_sqrt(const Fr &a, Fr &root) {
    if (a.is_zero()) { root = a; return true; }
    const Fr one = Fr::one();
    Fr w = a.pow(JJ_SQRT_EXP, 7);     // a^((t-1)/2)
    Fr x = a * w;                     // a^((t+1)/2): the root up to a 2^32-th root of unity
    Fr b = x * w;                     // a^t: its order is a power of two, <= 2^31 iff a is a square
    Fr z = fr_root_of_unity();
    int v = FR_TWO_ADICITY;
    while (b != one) {
        int k = 0;
        Fr b2k = b;
        do {                          // least k with b^(2^k) = 1
            b2k = b2k.sqr();
            if (++k == v) return false;   // order 2^v: a is not a square (only possible on the first pass)
        } while (b2k != one);
        Fr s = z;
        for (int j = 0; j < v - k - 1; j++) s = s.sqr();
        z = s.sqr();
        b = b * z;
        x = x * s;
        v = k;
    }
    root = x;
    return true;
}

struct Ext { Fr x, y, z, t; };       // extended twisted Edwards coordinates

ZK_DEV Ext ext_identity() { Ext p; p.x = Fr::zero(); p.y = Fr::one(); p.z = Fr::one(); p.t = Fr::zero(); return p; }
ZK_DEV bool ext_is_identity(const Ext &p) { return p.x.is_zero() && p.y == p.z; }   // (0 : Z : Z : 0)

// add-2008-hwcd-3 (a = -1, k = 2d): 8 products + 1 by the constant
ZK_DEV Ext ext_add(const Ext &p, const Ext &q, const Fr &d2) {
    Fr a = (p.y - p.x) * (q.y - q.x);
    Fr b = (p.y + p.x) * (q.y + q.x);
    Fr c = p.t * d2 * q.t;
    Fr d = (p.z * q.z).dbl();
    Fr e = b - a, f = d - c, g = d + c, h = b + a;
    Ext r;
    r.x = e * f; r.y = g * h; r.t = e * h; r.z = f * g;
    return r;
}
// dbl-2008-hwcd (a = -1): 4 products + 4 squares
ZK_DEV Ext ext_dbl(const Ext &p) {
    Fr a = p.x.sqr(), b = p.y.sqr(), c = p.z.sqr().dbl();
    Fr d = a.neg();
    Fr e = (p.x + p.y).sqr() - a - b;
    Fr g = d + b, f = g - c, h = d - b;
    Ext r;
    r.x = e * f; r.y = g * h; r.t = e * h; r.z = f * g;
    return r;
}
// [r_J] P, MSB-first double-and-add over the fixed 252-bit order
ZK_DEV Ext ext_mul_order(const Ext &p, const Fr &d2) {
    Ext acc = p;                                   // bit 251 is set
    for (int i = JJ_ORDER_BITS - 2; i >= 0; i--) {
        acc = ext_dbl(acc);
        if ((JJ_ORDER[i >> 5] >> (i & 31)) & 1) acc = ext_add(acc, p, d2);
    }
    return acc;
}

// Point::read of one 32-byte encoding given as 8 little-endian words, with no subgroup test (the Unknown order).  On JJ_OK,
// p = (x : y : 1 : xy) in Montgomery form; otherwise JJ_NOT_IN_FIELD or JJ_NOT_ON_CURVE and p is unset.
ZK_DEV int jubjub_read(const uint32_t *enc, Ext &p) {
    Fr yc;
#pragma unroll
    for (int i = 0; i < 8; i++) yc.l[i] = enc[i];
    const uint32_t sign = yc.l[7] >> 31;
    yc.l[7] &= 0x7fffffffu;
    if (!Fr::canonical_lt_mod(yc)) return JJ_NOT_IN_FIELD;
    const Fr one = Fr::one(), d2 = jj_d2();
    Fr y = Fr::from_canonical(yc);
    Fr y2 = y.sqr();
    // x^2 = (y^2 - 1) / (d y^2 + 1); 2 (d y^2 + 1) = 2d y^2 + 2 is inverted instead, and 2 is folded back into the numerator
    Fr den = y2 * d2 + one.dbl();
    Fr u = (y2 - one).dbl() * den.inverse();
    Fr x;
    if (!fr_sqrt(u, x)) return JJ_NOT_ON_CURVE;
    if ((x.to_canonical().l[0] & 1u) != sign) x = x.neg();   // 0 stays 0 (edwards.rs:143-145)
    p.x = x; p.y = y; p.z = one; p.t = x * y;
    return JJ_OK;
}

// Point::write (edwards.rs:190-206) of the affine point (x, y) in Montgomery form: canonical y, the parity of x in bit 255
ZK_DEV void jubjub_encode(const Fr &x, const Fr &y, uint32_t *enc) {
    const Fr yc = y.to_canonical();
    const uint32_t sign = x.to_canonical().l[0] & 1u;
#pragma unroll
    for (int i = 0; i < 8; i++) enc[i] = yc.l[i];
    enc[7] |= sign << 31;
}

// Point::read + as_prime_order + into_xy of one 32-byte encoding given as 8 little-endian words.  On JJ_OK, x / y are the
// canonical (non-Montgomery) coordinates; otherwise they are zero.
ZK_DEV int jubjub_into_xy(const uint32_t *enc, Fr &x_out, Fr &y_out) {
    x_out = Fr::zero(); y_out = Fr::zero();
    Ext p;
    const int s = jubjub_read(enc, p);
    if (s != JJ_OK) return s;
    if (!ext_is_identity(ext_mul_order(p, jj_d2()))) return JJ_NOT_PRIME_ORDER;
    x_out = p.x.to_canonical(); y_out = p.y.to_canonical();
    return JJ_OK;
}

}  // namespace zkjj
