// CPU unit-test harness of the PRODUCT's round decisions of zk_import_confidential_block / zk_import_assets_block
// (zero_chain_b200/csrc/import.cuh) compiled with ZK_HOST_EMUL: import.cu's run_rounds, pass for pass, as loops over the
// items (the decisions in reverse item order, so the order of the threads must not matter), with a model verifier in place
// of the state pass and the pairing check.  Checked by tests/test_host_emul_import.py against the Python drivers' loop.
// Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "import.cuh"
#include <string.h>
#include <vector>

using namespace zkimp;

// The model verifier: intended[k] is the verdict transfer k's proof gets against the balance it was made for, the one with
// exactly the chain's earlier intended passes applied.  Against any other balance it gets 0.  So a row's verdict is
// intended[k] when that is a failure, else 1 when every earlier applied transfer of its chain passes, else 0.
static uint8_t model_verdict(size_t k, const uint8_t *kind, const uint32_t *key_a, const uint8_t *intended, const uint8_t *applied) {
    if (intended[k] != 1) return intended[k];
    for (size_t q = 0; q < k; q++)
        if ((!kind || kind[q] == IMP_TRANSFER) && key_a[q] == key_a[k] && applied[q] == 1 && intended[q] != 1) return 0;
    return 1;
}

extern "C" {
// Runs the rounds; returns -1, the lowest transaction with a bad index or kind, or -2 when a gathered row or proof differs
// from what it should hold.  undecided: max_rounds * n_tx bytes, row r = the transactions verified in round r.
long long emu_import(size_t n_keys, size_t n_tx, const uint8_t *kind, const uint32_t *key_a, const uint32_t *key_b, const uint8_t *fixed,
                     const uint8_t *intended, uint8_t *verdicts, uint32_t *rounds, uint8_t *undecided, size_t max_rounds) {
    std::vector<uint8_t> applied(n_tx + 1), rv(n_tx + 1), rows(IMP_ROW * n_tx + 1), proofs(192 * n_tx + 1), bs(64 * n_tx + 1),
        round_rows(IMP_ROW * n_tx + 1), round_proofs(192 * n_tx + 1);
    std::vector<uint32_t> pos(n_tx + 1), idx(n_tx + 1), first_fail(n_keys + 1);
    uint32_t cnt[IMP_COUNTERS] = {0, 0, IMP_NONE, 0};
    for (size_t i = 0; i < rows.size(); i++) rows[i] = (uint8_t)(i * 7 + 1);
    for (size_t i = 0; i < proofs.size(); i++) proofs[i] = (uint8_t)(i * 13 + 5);
    *rounds = 0;
    for (size_t k = n_tx; k-- > 0;) imp_start(k, (uint32_t)n_keys, kind, key_a, key_b, fixed, verdicts, applied.data(), cnt);
    if (cnt[IMP_BAD] != IMP_NONE) return cnt[IMP_BAD];
    size_t m = cnt[IMP_TRANSFERS];
    for (unsigned r = 0;; r++) {
        // the state pass: each transfer's balance_sender, here a byte pattern of the transaction and the round
        for (size_t k = 0; k < n_tx; k++)
            for (int b = 0; b < 64; b++) bs[64 * k + b] = (uint8_t)(k * 3 + r * 11 + b);
        if (!m) break;
        if (r >= max_rounds) return -3;
        *rounds = r + 1;
        for (size_t k = n_tx; k-- > 0;) imp_flag(k, kind, verdicts, pos.data());
        uint32_t run = 0;
        for (size_t k = 0; k < n_tx; k++) { const uint32_t f = pos[k]; pos[k] = run; run += f; }
        if (run != m) return -2;
        for (size_t i = IMP_WORDS * n_tx; i-- > 0;)
            imp_gather(i, kind, verdicts, pos.data(), rows.data(), proofs.data(), bs.data(), idx.data(), round_rows.data(), round_proofs.data());
        for (size_t j = 0; j < m; j++) {
            const size_t k = idx[j];
            undecided[r * n_tx + k] = 1;
            for (int b = 0; b < IMP_ROW; b++) {
                const uint8_t want = b >= IMP_BS && b < IMP_BS + 64 ? bs[64 * k + b - IMP_BS] : rows[IMP_ROW * k + b];
                if (round_rows[IMP_ROW * j + b] != want) return -2;
            }
            if (memcmp(&round_proofs[192 * j], &proofs[192 * k], 192)) return -2;
            rv[j] = model_verdict(k, kind, key_a, intended, applied.data());
        }
        for (size_t a = 0; a < n_keys; a++) first_fail[a] = IMP_NONE;
        cnt[IMP_FAILS] = cnt[IMP_LEFT] = 0;
        for (size_t j = m; j-- > 0;) imp_fail(j, idx.data(), key_a, rv.data(), first_fail.data(), cnt);
        for (size_t j = m; j-- > 0;) imp_decide(j, idx.data(), key_a, rv.data(), first_fail.data(), verdicts, applied.data(), cnt);
        if (!cnt[IMP_FAILS]) break;
        m = cnt[IMP_LEFT];
    }
    return -1;
}

// imp_tx_points over n_tx rows
void emu_tx_points(size_t n_tx, const uint8_t *rows, uint8_t *tx_points) {
    for (size_t i = 32 * n_tx; i-- > 0;) imp_tx_points(i, rows, tx_points);
}
}
