// The scalar split of k_scale_points (groth16.cu): k = k1 * u^2 + k0 by plain shift-and-subtract division, u the BLS parameter.
// One thread runs it while its block's other warp runs the doubling chain; for k < 2^255 both k0 < u^2 < 2^128 and
// k1 < 2^255 / 2^127 = 2^128, so the chain stops at bit 127.  Plain integer code: the ZK_HOST_EMUL build checks it on the CPU
// (tests/host_emul/emul.cpp) against Python's divmod.
#pragma once
#include "field.cuh"

namespace zkglv {
// u^2 = 0xd201000000010000^2, little-endian 32-bit words
#define ZK_GLV_U2_INIT {0x00000000u, 0x00000001u, 0x0001a402u, 0xac45a401u}

// k: 8 little-endian words, k < 2^255 (bit 255 is not read).  k0 = k mod u^2, k1 = k div u^2, 4 words each.
ZK_DEV void split_u2(const uint32_t *k, uint32_t k0[4], uint32_t k1[4]) {
    const uint32_t dv[4] = ZK_GLV_U2_INIT;
    uint32_t rem[5] = {0, 0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
    for (int i = 254; i >= 0; i--) {
        for (int w = 4; w > 0; w--) rem[w] = (rem[w] << 1) | (rem[w - 1] >> 31);
        rem[0] = (rem[0] << 1) | ((k[i >> 5] >> (i & 31)) & 1);
        bool ge = rem[4] != 0;
        if (!ge) { ge = true; for (int w = 3; w >= 0; w--) { if (rem[w] != dv[w]) { ge = rem[w] > dv[w]; break; } } }
        if (ge) {
            uint64_t br = 0;
            for (int w = 0; w < 4; w++) { uint64_t x = (uint64_t)rem[w] - dv[w] - br; rem[w] = (uint32_t)x; br = (x >> 63) & 1; }
            rem[4] -= (uint32_t)br;
            if (i < 128) q[i >> 5] |= 1u << (i & 31);
        }
    }
    for (int w = 0; w < 4; w++) { k0[w] = rem[w]; k1[w] = q[w]; }
}
}  // namespace zkglv
