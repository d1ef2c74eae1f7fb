// CPU unit-test harness of the PRODUCT's anonymous-transfer functions in zero_chain_b200/csrc/tx_build.cuh, compiled with
// ZK_HOST_EMUL: the key table (anon_key_entry), the row status (anon_status), the row pass (anonymous_row), the ring
// positions (anon_position) and the left pass (anonymous_left), run in the order zk_anonymous_fields_batch runs them and
// checked against the Python oracle by tests/test_host_emul_anon_build.py.  Test infrastructure only — never linked into
// libzkb200.so.
#define ZK_HOST_EMUL 1
#include "tx_build.cuh"
#include <string.h>
#include <vector>

using namespace zktb;

extern "C" {
int emu_anon_position(int s, int t, int j) { return anon_position(s, t, j); }

// rings: n * 11 indices; positions: n * 2 bytes; fields: n * 864 bytes.  0, or 1 when g_epoch fails to read.
int emu_anon_fields(size_t n_keys, const uint8_t *keys, size_t n, const uint8_t *sks, const uint32_t *rings, const uint8_t *positions,
                    const uint32_t *amounts, const uint8_t *rs, const uint8_t *alphas, const uint8_t *g_epoch, uint8_t *fields, uint8_t *rsks,
                    uint8_t *dks, uint8_t *status) {
    static uint32_t table[TB_TABLE_WORDS];
    uint32_t g[8];
    memcpy(g, g_epoch, 32);
    Ext gp;
    if (read_prime_order(g, gp) != JJ_OK) return 1;
    for (int e = 0; e < TB_WINDOWS * TB_DIGITS; e++) tb_epoch_entry(gp, e, table + TB_ENTRY_WORDS * e);
    // the key pass: every key an in-range index names, once
    std::vector<uint8_t> named(n_keys, 0), key_status(n_keys, 0xEE);
    std::vector<uint32_t> niels(TB_ENTRY_WORDS * n_keys);
    for (size_t k = 0; k < TB_RING_IN * n; k++)
        if (rings[k] < n_keys) named[rings[k]] = 1;
    for (size_t k = 0; k < n_keys; k++) {
        if (!named[k]) continue;
        uint32_t w[8];
        memcpy(w, keys + 32 * k, 32);
        key_status[k] = (uint8_t)anon_key_entry(w, niels.data() + TB_ENTRY_WORDS * k);
    }
    // the row pass
    std::vector<uint32_t> scratch(8 * TB_ANON_SCRATCH_SLOTS * (n ? n : 1));
    for (size_t i = 0; i < n; i++) {
        uint32_t sk[8], r[8], al[8];
        memcpy(sk, sks + 32 * i, 32); memcpy(r, rs + 32 * i, 32); memcpy(al, alphas + 32 * i, 32);
        const int st = anon_status(positions[2 * i], positions[2 * i + 1], rings + TB_RING_IN * i, n_keys, key_status.data());
        anonymous_row(st, positions[2 * i], sk, amounts[i], r, al, table, scratch.data() + i, n, fields + 32 * TB_N_ANON_FIELDS * i, rsks + 32 * i,
                      dks + 32 * i);
        status[i] = (uint8_t)st;
    }
    // the left pass
    for (size_t k = 0; k < TB_RING_IN * n; k++) {
        const size_t i = k / TB_RING_IN;
        const int j = (int)(k % TB_RING_IN);
        if (status[i]) continue;
        uint32_t r[8];
        memcpy(r, rs + 32 * i, 32);
        const uint32_t idx = rings[k];
        anonymous_left(load_niels(niels.data() + TB_ENTRY_WORDS * idx), keys + 32 * idx, j, anon_position(positions[2 * i], positions[2 * i + 1], j),
                       amounts[i], r, fields + 32 * TB_N_ANON_FIELDS * i);
    }
    return 0;
}
}
