// CPU unit-test harness of the PRODUCT's ElGamal header (zero_chain_b200/csrc/elgamal.cuh) compiled with ZK_HOST_EMUL: the
// per-ciphertext stage, the chunked table build and the index, checked by tests/test_host_emul_elgamal.py against the
// Python and C oracles.  Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "elgamal.cuh"
#include <string.h>
#include <vector>

using namespace zkeg;

extern "C" {
// elgamal_stage for n ciphertexts in the layout of zk_elgamal_decrypt_batch; venc: n * 32 bytes (untouched unless EG_OK)
void emu_eg_stage(size_t n, const uint8_t *dks, const uint8_t *cts, const uint8_t *pending, uint8_t *venc, uint8_t *status) {
    for (size_t i = 0; i < n; i++) {
        uint32_t v[8];
        status[i] = (uint8_t)elgamal_stage(dks + 32 * i, cts + 64 * i, pending ? pending + 64 * i : nullptr, v);
        if (status[i] == EG_OK) memcpy(venc + 32 * i, v, 32);
    }
}
// the table's first n entries (n <= 2^20), one eg_table_chunk call per chunk as the device's threads make them
void emu_eg_table(uint32_t n, uint8_t *table) {
    std::vector<uint32_t> scratch(24 * (size_t)n), t(8 * (size_t)n);
    for (uint32_t c = 0; c * EG_CHUNK < n; c++) eg_table_chunk(c, n, scratch.data(), t.data());
    memcpy(table, t.data(), 32 * (size_t)n);
}
// an index of 2^log_slots slots over n 32-byte keys (inserted in the given order), then a lookup of each of the m probes:
// found[j] = the entry number or EG_EMPTY
void emu_eg_index(int log_slots, uint32_t n, const uint8_t *keys, const uint32_t *order, uint32_t m, const uint8_t *probes,
                  uint32_t *found) {
    const uint32_t mask = (1u << log_slots) - 1;
    std::vector<uint32_t> index(mask + 1, EG_EMPTY), table(8 * (size_t)n);
    memcpy(table.data(), keys, 32 * (size_t)n);
    for (uint32_t j = 0; j < n; j++) eg_index_insert(index.data(), mask, table.data() + 8 * (size_t)order[j], order[j]);
    for (uint32_t j = 0; j < m; j++) {
        uint32_t enc[8];
        memcpy(enc, probes + 32 * (size_t)j, 32);
        found[j] = eg_lookup(index.data(), mask, table.data(), enc);
    }
}
}
