// BLS12-381 G1 / G2 group arithmetic for the MSM kernels (device code, templated on the base field).
//
// Replaces the reference's Jacobian routines used inside bellman's multiexp:
//   core/pairing/src/bls12_381/ec.rs  add_assign_mixed 446-526, add_assign 356-444, double 296-354,
//   negate 528-532, into_affine 586-618, zero/is_zero 224-240
//   Fq2: core/pairing/src/bls12_381/fq2.rs mul 145-158 (Karatsuba), square 109-123, inverse 183-201
// The bucket accumulators use extended Jacobian ("XYZZ": x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2)
// coordinates: a mixed addition costs 8M + 2S instead of Jacobian's 7M + 4S and a full addition
// 12M + 2S.  Every result leaves the device as a canonical affine point, so the coordinate system
// cannot affect the bytes the caller sees — only the group law matters, and the exceptional cases
// the reference handles explicitly (P + P -> double, ec.rs:394-397/473-476; P + (-P) -> infinity;
// infinity operands, ec.rs:357-365/447-456) are handled here the same way.
#pragma once
#include "field.cuh"

struct Fq2 {
    Fq c0, c1;
    ZK_DEV static Fq2 zero() { Fq2 r; r.c0 = Fq::zero(); r.c1 = Fq::zero(); return r; }
    ZK_DEV static Fq2 one() { Fq2 r; r.c0 = Fq::one(); r.c1 = Fq::zero(); return r; }
    ZK_DEV bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    ZK_DEV bool operator==(const Fq2 &b) const { return c0 == b.c0 && c1 == b.c1; }
    ZK_DEV bool operator!=(const Fq2 &b) const { return !(*this == b); }
    ZK_DEV friend Fq2 operator+(const Fq2 &a, const Fq2 &b) { Fq2 r; r.c0 = a.c0 + b.c0; r.c1 = a.c1 + b.c1; return r; }
    ZK_DEV friend Fq2 operator-(const Fq2 &a, const Fq2 &b) { Fq2 r; r.c0 = a.c0 - b.c0; r.c1 = a.c1 - b.c1; return r; }
    ZK_DEV Fq2 dbl() const { Fq2 r; r.c0 = c0.dbl(); r.c1 = c1.dbl(); return r; }
    ZK_DEV Fq2 neg() const { Fq2 r; r.c0 = c0.neg(); r.c1 = c1.neg(); return r; }
    ZK_DEV Fq2 cneg(bool f) const { return f ? neg() : *this; }
    ZK_F2FN friend Fq2 operator*(const Fq2 &a, const Fq2 &b) {   // (a0 b0 - a1 b1) + (a0 b1 + a1 b0) u
        Fq aa = a.c0 * b.c0, bb = a.c1 * b.c1;
        Fq t = (a.c0 + a.c1) * (b.c0 + b.c1);
        Fq2 r; r.c1 = t - aa - bb; r.c0 = aa - bb; return r;
    }
    ZK_F2FN Fq2 sqr() const {   // (a0+a1)(a0-a1) + 2 a0 a1 u
        Fq ab = c0 * c1;
        Fq2 r; r.c0 = (c0 + c1) * (c0 - c1); r.c1 = ab.dbl(); return r;
    }
    ZK_DEV Fq2 inverse() const {
        Fq n = (c0.sqr() + c1.sqr()).inverse();
        Fq2 r; r.c0 = c0 * n; r.c1 = (c1 * n).neg(); return r;
    }
};

// Affine point as stored in HBM: x | y in Montgomery limbs (96 B for G1, 192 B for G2);
// the point at infinity is the all-zero pattern ((0,0) is not on either curve).
template <class F>
struct Affine {
    F x, y;
    ZK_DEV bool is_inf() const { return x.is_zero() && y.is_zero(); }
    ZK_DEV static Affine inf() { Affine r; r.x = F::zero(); r.y = F::zero(); return r; }
};

template <class F>
struct XYZZ {
    F x, y, zz, zzz;
    ZK_DEV static XYZZ inf() { XYZZ r; r.x = F::zero(); r.y = F::zero(); r.zz = F::zero(); r.zzz = F::zero(); return r; }
    ZK_DEV bool is_inf() const { return zz.is_zero(); }
    ZK_DEV static XYZZ from_affine(const Affine<F> &p) {
        XYZZ r;
        if (p.is_inf()) return inf();
        r.x = p.x; r.y = p.y; r.zz = F::one(); r.zzz = F::one(); return r;
    }
    ZK_DEV XYZZ neg() const { XYZZ r = *this; r.y = y.neg(); return r; }

    // The doubling formulas, always inlined.  add() and add_mixed() use these in their equal-points branch instead of calling
    // dbl() / dbl_affine(): where those are separate functions (the units that are not ZK_HOT) the callee reloads uniform
    // registers, and a call made by some lanes of a diverged warp overwrote the uniform memory descriptor that the other
    // lanes' loads in add() still used (k_ic_sum: "an illegal instruction was encountered" when one proof of a warp hit the
    // doubling branch).  Inlined, the whole branch is in one function and the register allocation sees every use.
    // 2 * (affine p)   (mdbl-2008-s-1)
    ZK_DEV static XYZZ dbl_affine_inl(const Affine<F> &p) {
        if (p.is_inf()) return inf();
        F u = p.y.dbl(), v = u.sqr(), w = u * v, s = p.x * v;
        F xx = p.x.sqr(), m = xx.dbl() + xx;
        XYZZ r;
        r.x = m.sqr() - s.dbl();
        r.y = m * (s - r.x) - w * p.y;
        r.zz = v; r.zzz = w;
        return r;
    }
    // 2 * this   (dbl-2008-s-1)
    ZK_DEV XYZZ dbl_inl() const {
        if (is_inf()) return *this;
        F u = y.dbl(), v = u.sqr(), w = u * v, s = x * v;
        F xx = x.sqr(), m = xx.dbl() + xx;
        XYZZ r;
        r.x = m.sqr() - s.dbl();
        r.y = m * (s - r.x) - w * y;
        r.zz = v * zz; r.zzz = w * zzz;
        return r;
    }
    ZK_PTFN static XYZZ dbl_affine(const Affine<F> &p) { return dbl_affine_inl(p); }
    ZK_PTFN XYZZ dbl() const { return dbl_inl(); }
    // this += affine p   (madd-2008-s), p optionally negated by the caller beforehand
    ZK_PTFN void add_mixed(const Affine<F> &p) {
        if (p.is_inf()) return;
        if (is_inf()) { x = p.x; y = p.y; zz = F::one(); zzz = F::one(); return; }
        F u2 = p.x * zz, s2 = p.y * zzz;
        F pp_ = u2 - x, r = s2 - y;
        if (pp_.is_zero()) {
            if (r.is_zero()) *this = dbl_affine_inl(p); else *this = inf();
            return;
        }
        F pp = pp_.sqr(), ppp = pp_ * pp, q = x * pp;
        F x3 = r.sqr() - ppp - q.dbl();
        y = r * (q - x3) - y * ppp;
        x = x3;
        zz = zz * pp; zzz = zzz * ppp;
    }
    // this += o   (add-2008-s)
    ZK_PTFN void add(const XYZZ &o) {
        if (o.is_inf()) return;
        if (is_inf()) { *this = o; return; }
        F u1 = x * o.zz, u2 = o.x * zz, s1 = y * o.zzz, s2 = o.y * zzz;
        F pp_ = u2 - u1, r = s2 - s1;
        if (pp_.is_zero()) {
            if (r.is_zero()) *this = dbl_inl(); else *this = inf();
            return;
        }
        F pp = pp_.sqr(), ppp = pp_ * pp, q = u1 * pp;
        F x3 = r.sqr() - ppp - q.dbl();
        y = r * (q - x3) - s1 * ppp;
        x = x3;
        zz = zz * o.zz * pp; zzz = zzz * o.zzz * ppp;
    }
    // canonical affine (one field inversion; into_affine, ec.rs:586-618)
    ZK_PTFN Affine<F> to_affine() const {
        if (is_inf()) return Affine<F>::inf();
        F zi = zzz.inverse();          // 1/ZZZ
        F zi2 = (zi * zz).sqr();       // (ZZ/ZZZ)^2 = 1/ZZ   (ZZ^3 = ZZZ^2)
        Affine<F> r; r.x = x * zi2; r.y = y * zi; return r;
    }
};

// k * P for a canonical 256-bit scalar k (8 LE u32 words), MSB-first double-and-add
template <class F>
ZK_PTFN XYZZ<F> scalar_mul(const XYZZ<F> &p, const uint32_t *k) {
    XYZZ<F> acc = XYZZ<F>::inf();
    bool started = false;
    for (int i = 255; i >= 0; i--) {
        if (started) acc = acc.dbl();
        if ((k[i >> 5] >> (i & 31)) & 1) { acc.add(p); started = true; }
    }
    return acc;
}

typedef Affine<Fq> G1Affine;
typedef Affine<Fq2> G2Affine;
typedef XYZZ<Fq> G1XYZZ;
typedef XYZZ<Fq2> G2XYZZ;
