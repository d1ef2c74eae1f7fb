// CPU unit-test harness of the PRODUCT's shared launch of zk_import_block (zero_chain_b200/csrc/import.cuh sections 2, 4,
// 5 and 7) compiled with ZK_HOST_EMUL: the sections' rows compacted at their offsets into one pair of round buffers, a
// model verifier over them, and each section's verdicts read back at its own offset, as import.cu's launch_round runs
// them, loops over the items in place of threads (the decisions in reverse item order).  Checked by
// tests/test_host_emul_block_import.py against one-section runs.  Test infrastructure only — never linked into
// libzkb200.so.
#define ZK_HOST_EMUL 1
#include "import.cuh"
#include <vector>

using namespace zkimp;

// a proof's bytes, made from its row so that a proof moved with the wrong row shows
static void make_proofs(size_t n, const uint8_t *rows, std::vector<uint8_t> &proofs) {
    proofs.assign(192 * n + 1, 0);
    for (size_t k = 0; k < n; k++)
        for (int b = 0; b < 192; b++) proofs[192 * k + b] = (uint8_t)(rows[IMP_ROW * k + b % IMP_ROW] ^ b);
}
static size_t prefix(std::vector<uint32_t> &c, size_t n) {
    uint32_t s = 0;
    for (size_t k = 0; k < n; k++) {
        const uint32_t v = c[k];
        c[k] = s;
        s += v;
    }
    return s;
}

extern "C" {
// One launch over S chain-keyed sections (kind NULL: transfers) and, behind them, one section of issues and transfers
// (ekind; its issues compacted with imp_compact, as the asset issues and destroys are).  Section s: n[s] transactions,
// chain keys key[s] < n_keys[s], rows[s] (IMP_ROW bytes each; byte 0 is the verdict the model verifier gives the row),
// verdict[s] (in: IMP_UNDECIDED or a decided byte; out) and applied[s] (out), counters cnt[2 s] (failures) and
// cnt[2 s + 1] (left undecided).  The issue section: ne transactions, ekind, erows, everdicts (out).  round_rows /
// round_proofs: the launch's buffers; off: the S + 1 offsets.  Returns the launch's rows.
size_t emu_block_launch(int S, const size_t *n, const size_t *n_keys, const uint32_t *const *key, const uint8_t *const *rows,
                        uint8_t *const *verdict, uint8_t *const *applied, uint32_t *cnt, size_t ne, const uint8_t *ekind,
                        const uint8_t *erows, uint8_t *everdicts, uint8_t *round_rows, uint8_t *round_proofs, size_t *off) {
    std::vector<std::vector<uint32_t>> pos(S), idx(S);
    std::vector<size_t> m(S);
    size_t total = 0;
    for (int s = 0; s < S; s++) {
        std::vector<uint8_t> proofs, bs(64 * n[s] + 1, 0);
        make_proofs(n[s], rows[s], proofs);
        pos[s].assign(n[s] + 1, 0);
        idx[s].assign(n[s] + 1, 0);
        for (size_t k = 0; k < n[s]; k++) imp_flag(k, nullptr, verdict[s], pos[s].data());
        m[s] = prefix(pos[s], n[s]);
        off[s] = total;
        for (size_t i = IMP_WORDS * n[s]; i-- > 0;)
            imp_gather(i, nullptr, verdict[s], pos[s].data(), rows[s], proofs.data(), bs.data(), idx[s].data(), round_rows, round_proofs,
                       total);
        total += m[s];
    }
    std::vector<uint32_t> epos(ne + 1, 0);
    std::vector<uint8_t> eproofs;
    make_proofs(ne, erows, eproofs);
    for (size_t k = 0; k < ne; k++) epos[k] = ekind[k] != IMP_TRANSFER;
    const size_t me = prefix(epos, ne);
    off[S] = total;
    for (size_t i = (IMP_ROW + 192) / 4 * ne; i-- > 0;)
        imp_compact(i, IMP_ROW, true, ekind, epos.data(), erows, eproofs.data(), round_rows, round_proofs, total);
    total += me;

    std::vector<uint8_t> rv(total + 1);
    for (size_t j = 0; j < total; j++) rv[j] = round_rows[IMP_ROW * j];          // the model verifier
    for (int s = 0; s < S; s++) {
        std::vector<uint32_t> first_fail(n_keys[s] + 1, IMP_NONE);
        cnt[2 * s] = cnt[2 * s + 1] = 0;
        for (size_t j = m[s]; j-- > 0;) imp_fail(j, idx[s].data(), key[s], rv.data(), first_fail.data(), cnt + 2 * s, off[s]);
        for (size_t j = m[s]; j-- > 0;)
            imp_decide(j, idx[s].data(), key[s], rv.data(), first_fail.data(), verdict[s], applied[s], cnt + 2 * s, off[s]);
    }
    for (size_t k = ne; k-- > 0;) imp_an_scatter(k, true, ekind, epos.data(), rv.data(), everdicts, off[S]);
    return total;
}
}
