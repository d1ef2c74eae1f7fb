// CPU unit-test harness of the PRODUCT's passes of zk_import_asset_calls (zero_chain_b200/csrc/import.cuh, section 6)
// compiled with ZK_HOST_EMUL: each pass of import.cu's asset_calls_run as a loop over its items, in reverse item order, so
// the order of the threads must not matter; zk_bal_prefix_sum is a plain exclusive sum.  Built twice by
// tests/test_host_emul_asset_calls.py: with the product's hash and capacity, and with ZK_IAS_HASH / ZK_IAS_CAPACITY
// overridden so that every key lands in one probe chain.  Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include <vector>

#include "import.cuh"

using namespace zkimp;

static void exclusive_sum(uint32_t *c, size_t n) {
    uint32_t s = 0;
    for (size_t i = 0; i < n; i++) {
        const uint32_t v = c[i];
        c[i] = s;
        s += v;
    }
}

extern "C" {
// Passes 1, 3 and 4 with the issue and destroy verdicts given (what pass 2's scatter leaves in verdicts).  The grown
// table's rows go to new_ids / new_keys / balances / pendings / slot_flags (room for n_slots + 2 n_tx rows; the first
// n_slots copied in), slot_a / slot_b and asset_ids per transaction; cnt: IMP_AS_COUNTERS words as the device leaves them
// after the second read.  The passes after a failing check run as on the device up to that read.
void emu_as_resolve(size_t n_slots, const uint32_t *slot_ids, const uint8_t *slot_keys, const uint8_t *balances_in, const uint8_t *pendings_in,
                    const uint8_t *flags_in, uint32_t next_id, uint8_t new_slot_flags, size_t n_tx, const uint8_t *kind, const uint32_t *asset_id,
                    const uint8_t *rows, const uint8_t *verdicts, uint32_t *asset_ids, uint32_t *slot_a, uint32_t *slot_b, uint32_t *new_ids,
                    uint8_t *new_keys, uint8_t *balances, uint8_t *pendings, uint8_t *slot_flags, uint32_t *cnt) {
    const size_t n_ref = 2 * n_tx, cap = ZK_IAS_CAPACITY(n_slots + n_ref);
    std::vector<uint32_t> table(cap, IMP_NONE), flag(n_tx + 1), ipos(n_tx + 1), ref_id(n_ref + 1), newpos(n_ref + 1);
    std::vector<uint8_t> ref_on(n_ref + 1);
    const ImpAsKeys t{slot_ids, slot_keys, ref_id.data(), rows, (uint32_t)n_slots};
    cnt[IMP_AS_FIXED] = cnt[IMP_AS_NEW] = 0;
    cnt[IMP_AS_BAD] = cnt[IMP_AS_DUP] = cnt[IMP_AS_OVF] = IMP_NONE;
    for (size_t k = n_tx; k-- > 0;) imp_as_start(k, kind, flag.data(), cnt);
    for (size_t r = n_slots; r-- > 0;) imp_as_row_insert(r, t, table.data(), (uint32_t)cap);
    for (size_t r = n_slots; r-- > 0;) imp_as_row_dup(r, t, table.data(), (uint32_t)cap, cnt);
    for (size_t k = n_tx; k-- > 0;) imp_as_issue_flag(k, kind, verdicts, ipos.data());
    exclusive_sum(ipos.data(), n_tx);
    for (size_t k = n_tx; k-- > 0;) imp_as_refs(k, next_id, kind, asset_id, verdicts, ipos.data(), asset_ids, ref_id.data(), ref_on.data(), cnt);
    for (size_t p = n_ref; p-- > 0;) imp_as_ref_insert(p, ref_on.data(), t, table.data(), (uint32_t)cap);
    for (size_t p = n_ref; p-- > 0;) imp_as_new(p, ref_on.data(), t, table.data(), (uint32_t)cap, newpos.data(), cnt);
    exclusive_sum(newpos.data(), n_ref);
    for (size_t r = 0; r < n_slots; r++) {
        new_ids[r] = slot_ids[r];
        for (int i = 0; i < 32; i++) new_keys[32 * r + i] = slot_keys[32 * r + i];
        for (int i = 0; i < 64; i++) balances[64 * r + i] = balances_in[64 * r + i], pendings[64 * r + i] = pendings_in[64 * r + i];
        slot_flags[r] = flags_in[r];
    }
    const uint8_t flags = (uint8_t)(new_slot_flags & ~3);
    for (size_t p = n_ref; p-- > 0;)
        imp_as_slot(p, ref_on.data(), t, table.data(), (uint32_t)cap, newpos.data(), flags, slot_a, slot_b, new_ids, new_keys, balances,
                    pendings, slot_flags);
}

// pass 2 around the verifier: the issue and destroy flags' sum, their compacted rows and proofs, and the scatter of rv
void emu_as_compact(size_t n_tx, const uint8_t *kind, const uint8_t *rows, const uint8_t *proofs, uint32_t *pos, uint32_t *cnt,
                    uint8_t *round_rows, uint8_t *round_proofs, const uint8_t *rv, uint8_t *verdicts) {
    cnt[IMP_AS_FIXED] = 0;
    cnt[IMP_AS_BAD] = IMP_NONE;
    for (size_t k = n_tx; k-- > 0;) imp_as_start(k, kind, pos, cnt);
    exclusive_sum(pos, n_tx);
    for (size_t i = IMP_WORDS * n_tx; i-- > 0;) imp_compact(i, IMP_ROW, true, kind, pos, rows, proofs, round_rows, round_proofs);
    for (size_t k = n_tx; k-- > 0;) imp_an_scatter(k, true, kind, pos, rv, verdicts);
}

void emu_as_tx_points(size_t n_tx, const uint8_t *kind, const uint8_t *rows, uint8_t *tx_points) {
    for (size_t i = 32 * n_tx; i-- > 0;) imp_as_tx_points(i, kind, rows, tx_points);
}
}
