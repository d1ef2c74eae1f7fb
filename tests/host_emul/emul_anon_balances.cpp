// CPU unit-test harness of the PRODUCT's anonymous-transfer header (zero_chain_b200/csrc/anon_balances.cuh, and the
// balances.cuh passes it reuses) compiled with ZK_HOST_EMUL: every pass of anon_balances.cu run as a loop over its items,
// in the same order of passes and with the same workspace layout, checked by tests/test_host_emul_anon_balances.py
// against the oracles.  Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "anon_balances.cuh"
#include <string.h>
#include <vector>

using namespace zkbal;

extern "C" {
// zk_balances_anonymous_block on host arrays; returns -1, or the lowest touched account that fails to decode
long long emu_anon_block(size_t n_acct, const uint8_t *keys, const uint8_t *balances, const uint8_t *pendings, const uint8_t *flags,
                         size_t n_tx, const uint32_t *members, const uint8_t *tx_points, const uint8_t *tx_extra, const uint8_t *g_epoch,
                         const uint8_t *applied, uint8_t *enc_balances, uint8_t *verify_points, uint8_t *status, uint8_t *new_balances,
                         uint8_t *new_pendings, uint8_t *new_flags) {
    const size_t ne = AN_RING * n_tx, ntp = AN_TX_POINTS * n_tx, nd = ntp + 4 * n_acct, np = 4 * n_acct;
    const size_t n_tiles = (ne + BAL_SORT_TILE - 1) / BAL_SORT_TILE;
    std::vector<uint32_t> keys0(ne + 1), keys1(ne + 1), vals0(ne + 1), vals1(ne + 1), hist(BAL_RADIX * n_tiles + 1), enc(8 * np + 8);
    std::vector<uint8_t> touched(n_acct + 1), recv_any(n_acct + 1), rflags(n_acct + 1), present(n_acct + 1), ok(nd + 1),
        has(2 * n_acct + 1), head(ne + 1);
    std::vector<Ext> dec(nd + 1), pts(np + 1);
    std::vector<Pair> delta(ne + 1), roll_b(n_acct + 1), roll_p(n_acct + 1), tot(2 * n_acct + 1);
    std::vector<Fr> prefix(np + 1);
    uint32_t bad = 0;
    const uint32_t na = (uint32_t)n_acct;
    for (size_t k = 0; k < n_tx; k++) an_touch(k, na, members, touched.data());
    for (size_t p = 0; p < nd; p++) an_decode(p, n_tx, tx_points, balances, pendings, flags, touched.data(), dec.data(), ok.data());
    for (size_t k = 0; k < n_tx; k++) an_tx(k, na, members, applied, dec.data(), ok.data(), keys0.data(), delta.data(), status, recv_any.data());
    for (size_t a = 0; a < n_acct; a++)
        bal_account(a, 0, flags, touched.data(), dec.data() + ntp, ok.data() + ntp, roll_b.data(), roll_p.data(), rflags.data(), &bad);
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
        // the elements in reverse: the order of the threads must not matter
        for (size_t j = ne; j-- > 0;) an_totals(j, ne, na, kin, vin, out[0].data(), delta.data(), tot.data(), has.data());
    }
    for (size_t a = 0; a < n_acct; a++)
        bal_acct_points(a, 0, na, touched.data(), roll_b.data(), roll_p.data(), rflags.data(), tot.data(), has.data(), recv_any.data(),
                        pts.data(), present.data());
    for (size_t c = 0; c * BAL_ENC_CHUNK < np; c++) bal_encode_chunk(c, np, pts.data(), prefix.data(), enc.data());
    for (size_t s = AN_VERIFY_POINTS * n_tx; s-- > 0;)
        an_finish_slot(s, members, status, keys, tx_points, tx_extra, g_epoch, enc.data(), enc_balances, verify_points);
    for (size_t a = 0; a < n_acct; a++)
        bal_finish_acct(a, 0, touched.data(), balances, pendings, flags, present.data(), enc.data(), new_balances, new_pendings, new_flags);
    return bad ? (long long)~bad : -1;
}
}
