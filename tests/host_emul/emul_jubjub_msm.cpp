// CPU unit-test harness of the PRODUCT's Jubjub MSM header (zero_chain_b200/csrc/jubjub_msm.cuh) compiled with
// ZK_HOST_EMUL: Niels negation, one bucket's accumulation, the bucket reduction of a window, Horner over windows and the
// per-entry stage of RedJubjub batch verification, checked against the Python oracle by
// tests/test_host_emul_jubjub_msm.py.  Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "jubjub_msm.cuh"
#include <string.h>

using namespace zkjm;

extern "C" {
// Point::read into Niels form (96 B); the status
int emu_jm_read_niels(const uint8_t *enc, uint32_t *niels) {
    uint32_t e[8];
    memcpy(e, enc, 32);
    Niels q;
    const int st = jm_read_niels(e, q);
    jm_niels_store(niels, q);
    return st;
}
void emu_jm_niels_cneg(const uint32_t *in, int neg, uint32_t *out) { jm_niels_store(out, jm_niels_cneg(jm_niels_load(in), neg != 0)); }
// Point::read into extended coordinates (128 B), for building buckets
int emu_jm_ext_read(const uint8_t *enc, uint32_t *ext) {
    uint32_t e[8];
    memcpy(e, enc, 32);
    Ext p;
    const int st = jubjub_read(e, p);
    if (st == JJ_OK) jm_ext_store(ext, p);
    return st;
}
void emu_jm_encode(const uint32_t *ext, uint8_t *out) {
    uint32_t e[8];
    jm_encode(jm_ext_load(ext), e);
    memcpy(out, e, 32);
}
void emu_jm_accumulate(const uint32_t *niels, const uint32_t *entries, uint32_t e0, uint32_t e1, uint32_t *ext) {
    jm_ext_store(ext, jm_accumulate(niels, entries, e0, e1));
}
void emu_jm_slice_sums(const uint32_t *buckets, uint32_t L, uint32_t *S, uint32_t *T) {
    Ext s, t;
    jm_slice_sums(buckets, L, s, t);
    jm_ext_store(S, s);
    jm_ext_store(T, t);
}
void emu_jm_window_sum(const uint32_t *S, const uint32_t *T, uint32_t n_slices, int log_L, uint32_t *out) {
    jm_ext_store(out, jm_window_sum(S, T, n_slices, log_L));
}
void emu_jm_horner(const uint32_t *R, int W, int c, uint32_t *out) { jm_ext_store(out, jm_horner(R, W, c)); }
// the per-entry stage for n entries (layout of zk_redjubjub_batch_verify): codes, z c per entry and the sum of z S
void emu_rj_batch_prep(size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *off, const uint8_t *zs,
                       uint8_t *codes, uint8_t *zc_out, uint8_t *zs_sum) {
    Fs sum = Fs::zero();
    for (size_t i = 0; i < n; i++) {
        uint32_t vk[8], sig[16], z[8];
        memcpy(vk, vks + 32 * i, 32);
        memcpy(sig, sigs + 64 * i, 64);
        memcpy(z, zs + 32 * i, 32);
        Niels nr, nvk;
        Fs zc, zsi;
        codes[i] = (uint8_t)rj_batch_entry(vk, sig, msgs + off[i], off[i + 1] - off[i], z, nr, nvk, zc, zsi);
        memcpy(zc_out + 32 * i, zc.l, 32);
        sum = sum + zsi;
    }
    memcpy(zs_sum, sum.l, 32);
}
}
