// Jubjub multi-scalar multiplication (sum_i s_i P_i over edwards::Point<Unknown>) and the per-entry stage of RedJubjub batch
// verification: the device arithmetic of jubjub_msm.cu.
//
// The MSM is Pippenger's, with the value-independent digit and sort kernels of msm.cuh (signed c-bit digits, one sort
// domain per window, entries grouped by bucket):
//   bases      each point once per call in Niels form (y - x, y + x, 2d x y), Montgomery Fr, 24 words; a negative digit
//              uses the negation, which swaps the first two and negates the third (jm_niels_cneg, a select, no branch)
//   buckets    one thread per bounded run of one bucket's entries: an extended-coordinate accumulator in registers and one
//              ext_madd (7 products) per entry; a bucket's runs are folded with ext_add
//   reduction  sum_d d B[d] per window over d = 1 .. 2^(c-1), organised for depth: the buckets are cut into slices of L; a
//              thread per slice keeps two running sums (jm_slice_sums), a thread per window folds the slices (jm_window_sum)
//   windows    Horner: R = sum_w 2^(c w) R_w
// The a = -1 twisted Edwards formulas are complete on Jubjub (d is not a square in Fr), so the identity, equal points,
// inverse points and small-order points need no special case anywhere.
//
// Everything is inlined into the kernels, like jubjub.cuh; thread-local arrays are only indexed with compile-time
// constants.  The same source compiles with ZK_HOST_EMUL for the CPU test (tests/host_emul/emul_jubjub_msm.cpp).
#pragma once
#include <stddef.h>
#include "redjubjub.cuh"

namespace zkjm {
using namespace zkjj;
using zkrj::Fs;
using zkrj::Niels;
using zkrj::ext_madd;
using zkrj::niels_of;

constexpr int JM_NIELS_WORDS = 24;     // 96 B per base
constexpr int JM_EXT_WORDS = 32;       // 128 B per bucket / partial
constexpr uint32_t JM_RUN = 16;        // most entries one accumulation thread adds

// ---- storage: Fr values as 8 consecutive words (16-byte aligned on the device: 128-bit loads) ---------------------------
ZK_DEV void jm_load_words(const uint32_t *src, uint32_t *w, int n16) {   // n16 groups of four words
#ifdef ZK_HOST_EMUL
    for (int k = 0; k < 4 * n16; k++) w[k] = src[k];
#else
#pragma unroll
    for (int k = 0; k < n16; k++) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(src) + k);
        w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
    }
#endif
}
ZK_DEV void jm_store_words(uint32_t *dst, const uint32_t *w, int n16) {
#ifdef ZK_HOST_EMUL
    for (int k = 0; k < 4 * n16; k++) dst[k] = w[k];
#else
#pragma unroll
    for (int k = 0; k < n16; k++) reinterpret_cast<uint4 *>(dst)[k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
#endif
}
ZK_DEV Niels jm_niels_load(const uint32_t *src) {
    uint32_t w[JM_NIELS_WORDS];
    jm_load_words(src, w, 6);
    Niels q;
#pragma unroll
    for (int i = 0; i < 8; i++) { q.ymx.l[i] = w[i]; q.ypx.l[i] = w[8 + i]; q.kt.l[i] = w[16 + i]; }
    return q;
}
ZK_DEV void jm_niels_store(uint32_t *dst, const Niels &q) {
    uint32_t w[JM_NIELS_WORDS];
#pragma unroll
    for (int i = 0; i < 8; i++) { w[i] = q.ymx.l[i]; w[8 + i] = q.ypx.l[i]; w[16 + i] = q.kt.l[i]; }
    jm_store_words(dst, w, 6);
}
ZK_DEV Ext jm_ext_load(const uint32_t *src) {
    uint32_t w[JM_EXT_WORDS];
    jm_load_words(src, w, 8);
    Ext p;
#pragma unroll
    for (int i = 0; i < 8; i++) { p.x.l[i] = w[i]; p.y.l[i] = w[8 + i]; p.z.l[i] = w[16 + i]; p.t.l[i] = w[24 + i]; }
    return p;
}
ZK_DEV void jm_ext_store(uint32_t *dst, const Ext &p) {
    uint32_t w[JM_EXT_WORDS];
#pragma unroll
    for (int i = 0; i < 8; i++) { w[i] = p.x.l[i]; w[8 + i] = p.y.l[i]; w[16 + i] = p.z.l[i]; w[24 + i] = p.t.l[i]; }
    jm_store_words(dst, w, 8);
}

// ---- bases ----------------------------------------------------------------------------------------------------------------
// neg ? -q : q.  -(x, y) = (-x, y): y - x and y + x trade places and 2d x y changes sign.
ZK_DEV Niels jm_niels_cneg(const Niels &q, bool neg) {
    const Fr kn = q.kt.neg();
    Niels r;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.ymx.l[i] = neg ? q.ypx.l[i] : q.ymx.l[i];
        r.ypx.l[i] = neg ? q.ymx.l[i] : q.ypx.l[i];
        r.kt.l[i] = neg ? kn.l[i] : q.kt.l[i];
    }
    return r;
}
// Point::read of one encoding (8 little-endian words) into Niels form; the identity's Niels form when it fails
ZK_DEV int jm_read_niels(const uint32_t *enc, Niels &q) {
    Ext p;
    const int st = jubjub_read(enc, p);
    q = st == JJ_OK ? niels_of(p.x, p.y, jj_d2()) : zkrj::niels_identity();
    return st;
}

// ---- buckets --------------------------------------------------------------------------------------------------------------
// The sum of the bases named by entries [e0, e1) of the bucket order: entry = base index | sign << 31
ZK_DEV Ext jm_accumulate(const uint32_t *niels, const uint32_t *entries, uint32_t e0, uint32_t e1) {
    Ext acc = ext_identity();
#pragma unroll 1
    for (uint32_t e = e0; e < e1; e++) {
        const uint32_t code = entries[e];
        const Niels q = jm_niels_load(niels + (size_t)JM_NIELS_WORDS * (code & 0x7fffffffu));
        acc = ext_madd(acc, jm_niels_cneg(q, code >> 31));
    }
    return acc;
}

// ---- reduction: sum_{d=1}^{N} d B[d] for one window -------------------------------------------------------------------
// Slice j holds the L buckets d = j L + 1 .. j L + L (B[d] stored at index d - 1).  Walking the slice from the top with a
// running sum T and a sum of running sums S gives S = sum_k k B[j L + k] and T = sum_k B[j L + k], 2 L additions.
ZK_DEV void jm_slice_sums(const uint32_t *buckets, uint32_t L, Ext &S, Ext &T) {
    const Fr d2 = jj_d2();
    S = ext_identity(); T = ext_identity();
#pragma unroll 1
    for (uint32_t k = L; k-- > 0;) {
        T = ext_add(T, jm_ext_load(buckets + (size_t)JM_EXT_WORDS * k), d2);
        S = ext_add(S, T, d2);
    }
}
// The window's sum from its slices: sum_j (S_j + j L T_j) = sum_j S_j + 2^log_L (sum_j j T_j), the inner sum again as
// running sums from the top.  S, T: n_slices points each.
ZK_DEV Ext jm_window_sum(const uint32_t *S, const uint32_t *T, uint32_t n_slices, int log_L) {
    const Fr d2 = jj_d2();
    Ext run = ext_identity(), acc = ext_identity();
#pragma unroll 1
    for (uint32_t j = n_slices; j-- > 1;) {
        run = ext_add(run, jm_ext_load(T + (size_t)JM_EXT_WORDS * j), d2);
        acc = ext_add(acc, run, d2);
    }
#pragma unroll 1
    for (int k = 0; k < log_L; k++) acc = ext_dbl(acc);
#pragma unroll 1
    for (uint32_t j = 0; j < n_slices; j++) acc = ext_add(acc, jm_ext_load(S + (size_t)JM_EXT_WORDS * j), d2);
    return acc;
}
// sum_w 2^(c w) R_w, Horner from the top window
ZK_DEV Ext jm_horner(const uint32_t *R, int W, int c) {
    const Fr d2 = jj_d2();
    Ext acc = jm_ext_load(R + (size_t)JM_EXT_WORDS * (W - 1));
#pragma unroll 1
    for (int w = W - 2; w >= 0; w--) {
#pragma unroll 1
        for (int k = 0; k < c; k++) acc = ext_dbl(acc);
        acc = ext_add(acc, jm_ext_load(R + (size_t)JM_EXT_WORDS * w), d2);
    }
    return acc;
}
// Point::write of an extended point
ZK_DEV void jm_encode(const Ext &p, uint32_t *enc) {
    const Fr zi = p.z.inverse();
    jubjub_encode(p.x * zi, p.y * zi, enc);
}

// ---- RedJubjub batch verification: one entry ---------------------------------------------------------------------------
// redjubjub::batch_verify's per-entry work for entry i (core/jubjub/src/redjubjub.rs:176-199) with the Diversifier generator,
// as multiexp terms: z R (base R, scalar z) and (z c) vk (base vk, scalar z c), plus z S, which the caller sums over the batch
// for the one -P_G term.  vk: 8 words; sig: 16 (rbar then sbar); z: 8, canonical.  Returns RJ_OK, or the entry's rejection
// in the per-signature order (RJ_BAD_VK, RJ_BAD_R, RJ_BAD_S); on a rejection the outputs are the identity and zero scalars,
// so the multiexp stays defined.  Scalars come out canonical: from_canonical(z) c = z R c / R = z c mod r_J.
ZK_DEV int rj_batch_entry(const uint32_t *vk, const uint32_t *sig, const uint8_t *msg, uint64_t mlen, const uint32_t *z, Niels &nr,
                          Niels &nvk, Fs &zc, Fs &zs) {
    Fs c;
    {
        uint64_t rbar[4], dg[8];
#pragma unroll
        for (int i = 0; i < 4; i++) rbar[i] = (uint64_t)sig[2 * i] | ((uint64_t)sig[2 * i + 1] << 32);
        zkrj::h_star_digest(rbar, msg, mlen, dg);
        c = zkrj::fs_to_uniform(dg);
    }
    nr = zkrj::niels_identity(); nvk = zkrj::niels_identity();
    zc = Fs::zero(); zs = Fs::zero();
    Niels a, r;
    if (jm_read_niels(vk, a) != JJ_OK) return zkrj::RJ_BAD_VK;
    if (jm_read_niels(sig, r) != JJ_OK) return zkrj::RJ_BAD_R;
    Fs s, zf;
#pragma unroll
    for (int i = 0; i < 8; i++) { s.l[i] = sig[8 + i]; zf.l[i] = z[i]; }
    if (!Fs::canonical_lt_mod(s)) return zkrj::RJ_BAD_S;
    zf = Fs::from_canonical(zf);
    nr = r; nvk = a;
    zc = zf * c;
    zs = zf * s;
    return zkrj::RJ_OK;
}

}  // namespace zkjm
