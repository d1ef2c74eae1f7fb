// CPU unit-test harness: compiles the PRODUCT's device headers (zero_chain_b200/csrc/*.cuh) with
// ZK_HOST_EMUL so the limb-level algorithms can be checked against the oracle without a GPU.
// Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "field.cuh"
#include <string.h>
extern "C" {
void emu_fq_mul(const uint32_t *a, const uint32_t *b, uint32_t *o) { Fq x, y; memcpy(x.l, a, 48); memcpy(y.l, b, 48); Fq r = x * y; memcpy(o, r.l, 48); }
void emu_fq_add(const uint32_t *a, const uint32_t *b, uint32_t *o) { Fq x, y; memcpy(x.l, a, 48); memcpy(y.l, b, 48); Fq r = x + y; memcpy(o, r.l, 48); }
void emu_fq_sub(const uint32_t *a, const uint32_t *b, uint32_t *o) { Fq x, y; memcpy(x.l, a, 48); memcpy(y.l, b, 48); Fq r = x - y; memcpy(o, r.l, 48); }
void emu_fq_neg(const uint32_t *a, uint32_t *o) { Fq x; memcpy(x.l, a, 48); Fq r = x.neg(); memcpy(o, r.l, 48); }
void emu_fq_inv(const uint32_t *a, uint32_t *o) { Fq x; memcpy(x.l, a, 48); Fq r = x.inverse(); memcpy(o, r.l, 48); }
void emu_fq_invf(const uint32_t *a, uint32_t *o) { Fq x; memcpy(x.l, a, 48); Fq r = x.inverse_fermat(); memcpy(o, r.l, 48); }
void emu_fq_from(const uint32_t *a, uint32_t *o) { Fq x; memcpy(x.l, a, 48); Fq r = Fq::from_canonical(x); memcpy(o, r.l, 48); }
void emu_fq_to(const uint32_t *a, uint32_t *o) { Fq x; memcpy(x.l, a, 48); Fq r = x.to_canonical(); memcpy(o, r.l, 48); }
int emu_fq_lt(const uint32_t *a) { Fq x; memcpy(x.l, a, 48); return Fq::canonical_lt_mod(x); }
void emu_fr_mul(const uint32_t *a, const uint32_t *b, uint32_t *o) { Fr x, y; memcpy(x.l, a, 32); memcpy(y.l, b, 32); Fr r = x * y; memcpy(o, r.l, 32); }
void emu_fr_add(const uint32_t *a, const uint32_t *b, uint32_t *o) { Fr x, y; memcpy(x.l, a, 32); memcpy(y.l, b, 32); Fr r = x + y; memcpy(o, r.l, 32); }
void emu_fr_sub(const uint32_t *a, const uint32_t *b, uint32_t *o) { Fr x, y; memcpy(x.l, a, 32); memcpy(y.l, b, 32); Fr r = x - y; memcpy(o, r.l, 32); }
void emu_fr_neg(const uint32_t *a, uint32_t *o) { Fr x; memcpy(x.l, a, 32); Fr r = x.neg(); memcpy(o, r.l, 32); }
void emu_fr_inv(const uint32_t *a, uint32_t *o) { Fr x; memcpy(x.l, a, 32); Fr r = x.inverse(); memcpy(o, r.l, 32); }
void emu_fr_invf(const uint32_t *a, uint32_t *o) { Fr x; memcpy(x.l, a, 32); Fr r = x.inverse_fermat(); memcpy(o, r.l, 32); }
void emu_fr_from(const uint32_t *a, uint32_t *o) { Fr x; memcpy(x.l, a, 32); Fr r = Fr::from_canonical(x); memcpy(o, r.l, 32); }
void emu_fr_to(const uint32_t *a, uint32_t *o) { Fr x; memcpy(x.l, a, 32); Fr r = x.to_canonical(); memcpy(o, r.l, 32); }
int emu_fr_lt(const uint32_t *a) { Fr x; memcpy(x.l, a, 32); return Fr::canonical_lt_mod(x); }
}

#include "curve.cuh"
template <class F> static void t_madd(const uint32_t *acc_aff, const uint32_t *p, uint32_t *o) {
    // (affine acc lifted to XYZZ, scaled by a non-trivial Z to exercise projective paths) + affine p
    Affine<F> a, b; memcpy(&a, acc_aff, sizeof(a)); memcpy(&b, p, sizeof(b));
    XYZZ<F> x = XYZZ<F>::from_affine(a);
    x = x.dbl(); x.add_mixed(b);            // 2a + b
    Affine<F> r = x.to_affine(); memcpy(o, &r, sizeof(r));
}
template <class F> static void t_add(const uint32_t *pa, const uint32_t *pb, uint32_t *o) {
    Affine<F> a, b; memcpy(&a, pa, sizeof(a)); memcpy(&b, pb, sizeof(b));
    XYZZ<F> x = XYZZ<F>::from_affine(a).dbl(), y = XYZZ<F>::from_affine(b).dbl();
    y.add_mixed(b);                         // 3b
    x.add(y);                               // 2a + 3b
    Affine<F> r = x.to_affine(); memcpy(o, &r, sizeof(r));
}
template <class F> static void t_plain_add(const uint32_t *pa, const uint32_t *pb, uint32_t *o, int mixed) {
    Affine<F> a, b; memcpy(&a, pa, sizeof(a)); memcpy(&b, pb, sizeof(b));
    XYZZ<F> x = XYZZ<F>::from_affine(a);
    if (mixed) x.add_mixed(b); else x.add(XYZZ<F>::from_affine(b));
    Affine<F> r = x.to_affine(); memcpy(o, &r, sizeof(r));
}
template <class F> static void t_mul(const uint32_t *pa, const uint32_t *k, uint32_t *o) {
    Affine<F> a; memcpy(&a, pa, sizeof(a));
    Affine<F> r = scalar_mul(XYZZ<F>::from_affine(a), k).to_affine(); memcpy(o, &r, sizeof(r));
}
extern "C" {
void emu_g1_2a_plus_b(const uint32_t *a, const uint32_t *b, uint32_t *o) { t_madd<Fq>(a, b, o); }
void emu_g2_2a_plus_b(const uint32_t *a, const uint32_t *b, uint32_t *o) { t_madd<Fq2>(a, b, o); }
void emu_g1_2a_plus_3b(const uint32_t *a, const uint32_t *b, uint32_t *o) { t_add<Fq>(a, b, o); }
void emu_g2_2a_plus_3b(const uint32_t *a, const uint32_t *b, uint32_t *o) { t_add<Fq2>(a, b, o); }
void emu_g1_add(const uint32_t *a, const uint32_t *b, uint32_t *o, int mixed) { t_plain_add<Fq>(a, b, o, mixed); }
void emu_g2_add(const uint32_t *a, const uint32_t *b, uint32_t *o, int mixed) { t_plain_add<Fq2>(a, b, o, mixed); }
void emu_g1_mul(const uint32_t *a, const uint32_t *k, uint32_t *o) { t_mul<Fq>(a, k, o); }
void emu_g2_mul(const uint32_t *a, const uint32_t *k, uint32_t *o) { t_mul<Fq2>(a, k, o); }
}

// ---- batched-affine pair additions (msm_batchaff.cuh, msm_affine_core.cuh): the per-pair classification / finish functions and the
// simultaneous-inversion walk, replayed on the host for ONE bucket of n points -> ceil(n/2) points
#include <vector>
#include "msm_affine_core.cuh"
template <class F> static void t_batch_pairs(const uint32_t *in, int n, uint32_t *out) {
    using namespace zkmsm;
    std::vector<Affine<F>> p(n);
    memcpy(p.data(), in, sizeof(Affine<F>) * n);
    int m = (n + 1) / 2;
    std::vector<F> scratch(m);
    std::vector<Affine<F>> o(m);
    F run = F::one();
    for (int j = 0; j < m; j++) {
        bool has1 = 2 * j + 1 < n;
        Affine<F> p0 = p[2 * j], p1 = has1 ? p[2 * j + 1] : Affine<F>::inf();
        F den; pair_classify(p0, p1, has1, den);
        scratch[j] = run; run = run * den;
    }
    F inv = run.inverse();
    for (int j = m - 1; j >= 0; j--) {
        bool has1 = 2 * j + 1 < n;
        Affine<F> p0 = p[2 * j], p1 = has1 ? p[2 * j + 1] : Affine<F>::inf();
        F den; int mode = pair_classify(p0, p1, has1, den);
        F dinv = inv * scratch[j]; inv = inv * den;
        o[j] = pair_finish(mode, p0, p1, dinv);
    }
    memcpy(out, o.data(), sizeof(Affine<F>) * m);
}
extern "C" {
void emu_g1_batch_pairs(const uint32_t *in, int n, uint32_t *out) { t_batch_pairs<Fq>(in, n, out); }
void emu_g2_batch_pairs(const uint32_t *in, int n, uint32_t *out) { t_batch_pairs<Fq2>(in, n, out); }
}

#include "field_wide.cuh"
extern "C" {
void emu_fq_mul_sep(const uint32_t *a, const uint32_t *b, uint32_t *o) { Fq x, y; memcpy(x.l, a, 48); memcpy(y.l, b, 48); Fq r = zkwide::mul_sep(x, y); memcpy(o, r.l, 48); }
void emu_fq_sqr_sep(const uint32_t *a, uint32_t *o) { Fq x; memcpy(x.l, a, 48); Fq r = zkwide::sqr_sep(x); memcpy(o, r.l, 48); }
void emu_fq_mul_sub_mul(const uint32_t *a, const uint32_t *b, const uint32_t *c, const uint32_t *d, uint32_t *o) {
    Fq x, y, z, w; memcpy(x.l, a, 48); memcpy(y.l, b, 48); memcpy(z.l, c, 48); memcpy(w.l, d, 48);
    Fq r = zkwide::mul_sub_mul(x, y, z, w); memcpy(o, r.l, 48);
}
}

// ---- the scalar split of k_scale_points (glv_split.cuh): n scalars of 8 words -> k0 | k1, 4 words each
#include <stddef.h>
#include "glv_split.cuh"
extern "C" void emu_glv_split_many(const uint32_t *k, size_t n, uint32_t *out) {
    for (size_t i = 0; i < n; i++) zkglv::split_u2(k + 8 * i, out + 8 * i, out + 8 * i + 4);
}
