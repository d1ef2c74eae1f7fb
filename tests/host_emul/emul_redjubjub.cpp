// CPU unit-test harness of the PRODUCT's RedJubjub header (zero_chain_b200/csrc/redjubjub.cuh) compiled with ZK_HOST_EMUL:
// BLAKE2b (H* before the reduction), Fs::to_uniform and whole verifications, checked against the Python oracle by
// tests/test_host_emul_redjubjub.py.  Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "redjubjub.cuh"
#include <string.h>

using namespace zkrj;

extern "C" {
// the 64-byte BLAKE2b digest of rbar (32 B) || msg with the H* personalization
void emu_rj_h_star_digest(const uint8_t *rbar, const uint8_t *msg, uint64_t mlen, uint8_t *out) {
    uint64_t r[4], h[8];
    memcpy(r, rbar, 32);                 // little-endian host: the byte order of the words
    h_star_digest(r, msg, mlen, h);
    memcpy(out, h, 64);
}
// Fs::to_uniform of a 64-byte digest -> 32 bytes, canonical little-endian
void emu_rj_to_uniform(const uint8_t *digest, uint8_t *out) {
    uint64_t d[8];
    memcpy(d, digest, 64);
    Fs c = fs_to_uniform(d);
    memcpy(out, c.l, 32);
}
// n signatures in the layout of zk_redjubjub_verify_batch
void emu_rj_verify(size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *off, uint8_t *verdicts) {
    for (size_t i = 0; i < n; i++) {
        uint32_t vk[8], sig[16];
        memcpy(vk, vks + 32 * i, 32);
        memcpy(sig, sigs + 64 * i, 64);
        verdicts[i] = (uint8_t)redjubjub_verify(vk, sig, msgs + off[i], off[i + 1] - off[i]);
    }
}
}
