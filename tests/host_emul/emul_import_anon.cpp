// CPU unit-test harness of the PRODUCT's passes of zk_import_anonymous_block (zero_chain_b200/csrc/import.cuh, section 5)
// compiled with ZK_HOST_EMUL: each pass of import.cu's anon_run as a loop over its items, in reverse item order, so the
// order of the threads must not matter.  Checked by tests/test_host_emul_import_anon.py against AnonIssueTx.verify_points,
// the Python driver's index checks and a numpy restatement.  Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "import.cuh"

using namespace zkimp;

extern "C" {
// imp_an_start over n_tx transactions; cnt: IMP_COUNTERS words, returned as the device leaves them
void emu_an_start(size_t n_tx, uint32_t n_acct, int issues_ok, const uint8_t *kind, const uint32_t *members, uint32_t *flag, uint32_t *cnt) {
    cnt[IMP_ISSUES] = cnt[IMP_TRANSFERS] = 0;
    cnt[IMP_BAD] = IMP_NONE;
    for (size_t k = n_tx; k-- > 0;) imp_an_start(k, n_acct, issues_ok != 0, kind, members, flag, cnt);
}

void emu_an_issue_rows(size_t n_tx, const uint8_t *kind, const uint32_t *pos, const uint8_t *keys, const uint32_t *members,
                       const uint8_t *tx_points, const uint8_t *issue_fields, const uint8_t *tx_extra, const uint8_t *g_epoch,
                       const uint8_t *proofs, uint8_t *rows, uint8_t *round_proofs) {
    for (size_t i = IMP_AN_ISSUE_WORDS * n_tx; i-- > 0;)
        imp_an_issue_row(i, kind, pos, keys, members, tx_points, issue_fields, tx_extra, g_epoch, proofs, rows, round_proofs);
}

void emu_an_scatter(size_t n_tx, int issues, const uint8_t *kind, const uint32_t *pos, const uint8_t *rv, uint8_t *verdicts) {
    for (size_t k = n_tx; k-- > 0;) imp_an_scatter(k, issues != 0, kind, pos, rv, verdicts);
}

void emu_an_gather(size_t n_tx, const uint8_t *kind, const uint32_t *pos, const uint8_t *verify_points, const uint8_t *proofs,
                   uint8_t *rows, uint8_t *round_proofs) {
    for (size_t i = IMP_AN_WORDS * n_tx; i-- > 0;) imp_an_gather(i, kind, pos, verify_points, proofs, rows, round_proofs);
}
}
