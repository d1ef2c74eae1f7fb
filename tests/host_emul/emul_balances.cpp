// CPU unit-test harness of the PRODUCT's balance-update header (zero_chain_b200/csrc/balances.cuh) compiled with
// ZK_HOST_EMUL: every pass of balances.cu run as a loop over its items, in the same order of passes and with the same
// workspace layout, checked by tests/test_host_emul_balances.py against the Python oracle.  Test infrastructure only —
// never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "balances.cuh"
#include <string.h>
#include <vector>

using namespace zkbal;

extern "C" {
// zk_balances_confidential_block on host arrays; returns -1, or the lowest touched account that fails to decode
long long emu_bal_block(size_t n_acct, const uint8_t *balances, const uint8_t *pendings, const uint8_t *flags, size_t n_tx,
                        const uint32_t *sender, const uint32_t *recipient, const uint8_t *tx_points, const uint8_t *applied,
                        uint8_t *balance_sender, uint8_t *balance_after, uint8_t *status, uint8_t *new_balances, uint8_t *new_pendings,
                        uint8_t *new_flags) {
    const size_t ne = 2 * n_tx, np = 4 * n_tx + 4 * n_acct, n_tiles = (ne + BAL_SORT_TILE - 1) / BAL_SORT_TILE;
    std::vector<uint32_t> keys0(ne + 1), keys1(ne + 1), vals0(ne + 1), vals1(ne + 1), hist(BAL_RADIX * n_tiles + 1), enc(8 * np + 8);
    std::vector<uint8_t> touched(n_acct + 1), recv_any(n_acct + 1), rflags(n_acct + 1), present(n_acct + 1), ok(np + 1),
        has(2 * n_acct + 1), head(ne + 1);
    std::vector<Ext> dec(np + 1), pts(np + 1);
    std::vector<Pair> delta(ne + 1), roll_b(n_acct + 1), roll_p(n_acct + 1), tot(2 * n_acct + 1);
    std::vector<Fr> prefix(np + 1);
    uint32_t bad = 0;
    const uint32_t na = (uint32_t)n_acct;
    for (size_t k = 0; k < n_tx; k++) bal_touch(k, na, sender, recipient, keys0.data(), touched.data());
    for (size_t p = 0; p < np; p++) bal_decode(p, n_tx, tx_points, balances, pendings, flags, touched.data(), dec.data(), ok.data());
    for (size_t k = 0; k < n_tx; k++) bal_tx(k, na, sender, recipient, applied, dec.data(), ok.data(), delta.data(), status, recv_any.data());
    for (size_t a = 0; a < n_acct; a++) bal_account(a, n_tx, flags, touched.data(), dec.data(), ok.data(), roll_b.data(), roll_p.data(), rflags.data(), &bad);
    if (n_tx) {
        int bits = 0;
        while (bits < 32 && ((2 * (uint64_t)n_acct) >> bits)) bits++;
        const int passes = bits <= BAL_RADIX_BITS ? 1 : (bits + BAL_RADIX_BITS - 1) / BAL_RADIX_BITS;
        uint32_t *kin = keys0.data(), *vin = nullptr, *kout = keys1.data(), *vout = vals1.data();
        for (int p = 0; p < passes; p++) {
            std::fill(hist.begin(), hist.end(), 0);
            // the tiles run in reverse: the order of the threads must not matter
            for (size_t t = n_tiles; t-- > 0;) bal_radix_hist(t, ne, kin, BAL_RADIX_BITS * p, n_tiles, hist.data());
            uint32_t run = 0;
            for (size_t i = 0; i < BAL_RADIX * n_tiles; i++) { const uint32_t v = hist[i]; hist[i] = run; run += v; }
            for (size_t t = n_tiles; t-- > 0;) bal_radix_scatter(t, ne, kin, vin, BAL_RADIX_BITS * p, n_tiles, hist.data(), kout, vout);
            kin = kout; vin = vout;
            kout = kin == keys1.data() ? keys0.data() : keys1.data();
            vout = vin == vals1.data() ? vals0.data() : vals1.data();
        }
        for (size_t j = 0; j < ne; j++) bal_heads(j, kin, head.data());
        std::vector<size_t> ln(1, ne);
        std::vector<std::vector<Pair>> agg(1), out(1, std::vector<Pair>(ne + 1));
        std::vector<std::vector<uint8_t>> hd(1, head);
        for (size_t n = ne; n > BAL_SCAN_CHUNK;) {
            n = (n + BAL_SCAN_CHUNK - 1) / BAL_SCAN_CHUNK;
            ln.push_back(n); agg.emplace_back(n + 1); out.emplace_back(n + 1); hd.emplace_back(n + 1);
        }
        const size_t L = ln.size();
        for (size_t l = 0; l + 1 < L; l++)
            for (size_t c = 0; c < ln[l + 1]; c++)
                bal_scan_up(c, ln[l], l ? agg[l].data() : delta.data(), l ? nullptr : vin, hd[l].data(), agg[l + 1].data(), hd[l + 1].data());
        for (size_t l = L; l-- > 0;)
            for (size_t c = 0; c * BAL_SCAN_CHUNK < ln[l]; c++)
                bal_scan_down(c, ln[l], l ? agg[l].data() : delta.data(), l ? nullptr : vin, hd[l].data(),
                              l + 1 < L ? out[l + 1].data() : nullptr, l == 0, out[l].data());
        for (size_t j = 0; j < ne; j++)
            bal_tx_points(j, ne, na, kin, vin, out[0].data(), delta.data(), roll_b.data(), rflags.data(), status, pts.data(), tot.data(), has.data());
    }
    for (size_t a = 0; a < n_acct; a++)
        bal_acct_points(a, n_tx, na, touched.data(), roll_b.data(), roll_p.data(), rflags.data(), tot.data(), has.data(), recv_any.data(),
                        pts.data(), present.data());
    for (size_t c = 0; c * BAL_ENC_CHUNK < np; c++) bal_encode_chunk(c, np, pts.data(), prefix.data(), enc.data());
    for (size_t k = 0; k < n_tx; k++) bal_finish_tx(k, status, enc.data(), balance_sender, balance_after);
    for (size_t a = 0; a < n_acct; a++)
        bal_finish_acct(a, n_tx, touched.data(), balances, pendings, flags, present.data(), enc.data(), new_balances, new_pendings, new_flags);
    return bad ? (long long)~bad : -1;
}
}
