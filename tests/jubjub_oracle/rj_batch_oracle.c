/* TEST INFRASTRUCTURE (oracle) — redjubjub::batch_verify with the Diversifier generator, in plain C99 + OpenMP.  Not part of
 * the product; the tests and tools/redjubjub_batch_bench.py build it through tests/jubjub_oracle/rjb_coracle.py.
 *
 * It includes the RedJubjub oracle (redjubjub_oracle.c) as it is, for Point::read, BLAKE2b, Fs, P_G and the group law, and
 * adds the reference's batch loop (core/jubjub/src/redjubjub.rs:166-204): each entry z R + (z c) vk + (-(z S)) P_G by three
 * double-and-adds.  The entries are split over the OpenMP threads and their terms summed; it is the host-core baseline of
 * the device batch check. */
#include "redjubjub_oracle.c"
#include <stdlib.h>

/* zs: n * 32 B canonical randomizers.  *verdict and *first_bad as zk_redjubjub_batch_verify: the reference's early
 * `return false` becomes the lowest rejected index (first_bad = n when none is rejected). */
EXPORT void rjo_batch_verify(size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *off,
                             const uint8_t *zs, uint8_t *verdict, uint64_t *first_bad) {
    long long nn = (long long)n;
    uint8_t *code = (uint8_t *)calloc(n ? n : 1, 1);
    ext_t total;
    ext_zero(&total);
#pragma omp parallel
    {
        fr_t d2; jj_d2(&d2);
        ext_t acc; ext_zero(&acc);
#pragma omp for schedule(dynamic, 16)
        for (long long i = 0; i < nn; i++) {
            const uint8_t *sig = sigs + 64 * i;
            ext_t a, r, t;
            uint64_t s[4], c[4], z[4], w[4];
            if (read_point(vks + 32 * i, &a)) { code[i] = 2; continue; }
            if (read_point(sig, &r)) { code[i] = 3; continue; }
            load_le(s, sig + 32, 4);
            if (fs_raw_geq(s, JJ_ORDER)) { code[i] = 4; continue; }
            h_star(c, sig, 32, msgs + off[i], off[i + 1] - off[i]);
            load_le(z, zs + 32 * i, 4);
            fs_t fs_, fz, fc;
            fs_set_zero(&fs_); fs_set_zero(&fz); fs_set_zero(&fc);
            fs_from_repr(&fs_, s); fs_from_repr(&fz, z); fs_from_repr(&fc, c);
            fs_mul(&fs_, &fs_, &fz); fs_neg(&fs_, &fs_);
            fs_mul(&fc, &fc, &fz);
            ext_mul(&t, &r, z); ext_add(&acc, &acc, &t, &d2);
            fs_into_repr(w, &fc); ext_mul(&t, &a, w); ext_add(&acc, &acc, &t, &d2);
            fs_into_repr(w, &fs_); ext_pg(&t); ext_mul(&t, &t, w); ext_add(&acc, &acc, &t, &d2);
        }
#pragma omp critical
        ext_add(&total, &total, &acc, &d2);
    }
    *first_bad = n;
    *verdict = 1;
    for (size_t i = 0; i < n; i++)
        if (code[i]) { *verdict = code[i]; *first_bad = i; break; }
    free(code);
    if (*verdict != 1) return;
    for (int i = 0; i < 3; i++) ext_dbl(&total, &total);
    *verdict = (uint8_t)(fr_is_zero(&total.x) && fr_eq(&total.y, &total.z));
}
