// CPU unit-test harness of the PRODUCT's issue passes of zk_anonymous_calls_block (zero_chain_b200/csrc/anon_balances.cuh,
// and the balances.cuh passes it reuses) compiled with ZK_HOST_EMUL: every pass of anon_balances.cu's run_block with a
// kind array, run as a loop over its items, in the same order of passes and with the same workspace layout, checked by
// tests/test_host_emul_anon_issue.py against the oracles.  Test infrastructure only — never linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "anon_balances.cuh"
#include <string.h>
#include <algorithm>
#include <vector>

using namespace zkbal;

// zk_bal_sort: stable LSD radix sort of n keys (each <= 2 n_acct) by bal_radix_hist / bal_radix_scatter, the tiles in
// reverse (the order of the threads must not matter); returns the sorted keys and ids
static void radix_sort(size_t n, size_t n_acct, std::vector<uint32_t> &keys0, std::vector<uint32_t> &keys1, std::vector<uint32_t> &vals0,
                       std::vector<uint32_t> &vals1, const uint32_t **keys, const uint32_t **vals) {
    const size_t n_tiles = (n + BAL_SORT_TILE - 1) / BAL_SORT_TILE;
    std::vector<uint32_t> hist(BAL_RADIX * n_tiles + 1);
    int bits = 0;
    while (bits < 32 && ((2 * (uint64_t)n_acct) >> bits)) bits++;
    const int passes = bits <= BAL_RADIX_BITS ? 1 : (bits + BAL_RADIX_BITS - 1) / BAL_RADIX_BITS;
    uint32_t *kin = keys0.data(), *vin = nullptr, *kout = keys1.data(), *vout = vals1.data();
    for (int p = 0; p < passes; p++) {
        std::fill(hist.begin(), hist.end(), 0);
        for (size_t t = n_tiles; t-- > 0;) bal_radix_hist(t, n, kin, BAL_RADIX_BITS * p, n_tiles, hist.data());
        uint32_t run = 0;
        for (size_t i = 0; i < BAL_RADIX * n_tiles; i++) { const uint32_t v = hist[i]; hist[i] = run; run += v; }
        for (size_t t = n_tiles; t-- > 0;) bal_radix_scatter(t, n, kin, vin, BAL_RADIX_BITS * p, n_tiles, hist.data(), kout, vout);
        kin = kout; vin = vout;
        kout = kin == keys1.data() ? keys0.data() : keys1.data();
        vout = vin == vals1.data() ? vals0.data() : vals1.data();
    }
    *keys = kin;
    *vals = vin;
}

extern "C" {
// zk_anonymous_calls_block on host arrays (n_tx > 0); returns -1, or the lowest touched account that fails to decode
long long emu_anon_calls_block(size_t n_acct, const uint8_t *keys, const uint8_t *balances, const uint8_t *pendings, const uint8_t *flags,
                               size_t n_tx, const uint8_t *kind, const uint32_t *members, const uint8_t *tx_points, const uint8_t *tx_extra,
                               const uint8_t *g_epoch, const uint8_t *applied, uint8_t *enc_balances, uint8_t *verify_points,
                               uint8_t *issued, uint8_t *status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags) {
    const size_t ne = AN_RING * n_tx, ntp = AN_TX_POINTS * n_tx, nd = ntp + 4 * n_acct, np = 4 * n_acct + 2 * n_tx;
    std::vector<uint32_t> keys0(ne + 1), keys1(ne + 1), vals0(ne + 1), vals1(ne + 1), enc(8 * np + 8);
    std::vector<uint32_t> ikeys0(n_tx + 1), ikeys1(n_tx + 1), ivals0(n_tx + 1), ivals1(n_tx + 1), first(n_acct + 1, AN_NONE),
        fin(n_acct + 1), rd(ne + 1);
    std::vector<uint8_t> touched(n_acct + 1), recv_any(n_acct + 1), rflags(n_acct + 1), present(n_acct + 1), ok(nd + 1),
        has(2 * n_acct + 1), head(ne + 1);
    std::vector<Ext> dec(nd + 1), pts(np + 1);
    std::vector<Pair> delta(ne + 1), roll_b(n_acct + 1), roll_p(n_acct + 1), tot(2 * n_acct + 1);
    std::vector<Fr> prefix(np + 1);
    uint32_t bad = 0;
    const uint32_t na = (uint32_t)n_acct;
    for (size_t k = n_tx; k-- > 0;) an_call_touch(k, na, kind, members, touched.data(), first.data());
    for (size_t p = 0; p < nd; p++) an_decode(p, n_tx, tx_points, balances, pendings, flags, touched.data(), dec.data(), ok.data(), kind);
    for (size_t k = 0; k < n_tx; k++)
        an_call_tx(k, na, kind, members, applied, dec.data(), ok.data(), keys0.data(), delta.data(), status, recv_any.data(), ikeys0.data(),
                   pts.data() + 4 * n_acct);
    const uint32_t *iskeys, *isvals;
    radix_sort(n_tx, n_acct, ikeys0, ikeys1, ivals0, ivals1, &iskeys, &isvals);
    for (size_t a = 0; a < n_acct; a++)
        an_issue_account(a, n_tx, flags, touched.data(), first.data(), iskeys, isvals, dec.data(), ok.data(), roll_b.data(), roll_p.data(),
                         rflags.data(), fin.data(), &bad);
    const uint32_t *skeys, *svals;
    radix_sort(ne, n_acct, keys0, keys1, vals0, vals1, &skeys, &svals);
    for (size_t j = 0; j < ne; j++) bal_heads(j, skeys, head.data());
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
            bal_scan_up(c, ln[l], l ? agg[l].data() : delta.data(), l ? nullptr : svals, hd[l].data(), agg[l + 1].data(), hd[l + 1].data());
    for (size_t l = L; l-- > 0;)
        for (size_t c = 0; c * BAL_SCAN_CHUNK < ln[l]; c++)
            bal_scan_down(c, ln[l], l ? agg[l].data() : delta.data(), l ? nullptr : svals, hd[l].data(),
                          l + 1 < L ? out[l + 1].data() : nullptr, l == 0, out[l].data());
    for (size_t j = ne; j-- > 0;) an_totals(j, ne, na, skeys, svals, out[0].data(), delta.data(), tot.data(), has.data());
    for (size_t a = 0; a < n_acct; a++)
        bal_acct_points(a, 0, na, touched.data(), roll_b.data(), roll_p.data(), rflags.data(), tot.data(), has.data(), recv_any.data(),
                        pts.data(), present.data());
    for (size_t e = ne; e-- > 0;) an_issue_read(e, na, n_tx, kind, status, members, first.data(), iskeys, isvals, rd.data());
    for (size_t c = 0; c * BAL_ENC_CHUNK < np; c++) bal_encode_chunk(c, np, pts.data(), prefix.data(), enc.data());
    for (size_t s = AN_VERIFY_POINTS * n_tx; s-- > 0;)
        an_finish_slot(s, members, status, keys, tx_points, tx_extra, g_epoch, enc.data(), enc_balances, verify_points, kind, rd.data());
    for (size_t k = 0; k < n_tx; k++) an_issued(k, na, kind, status, enc.data(), issued);
    for (size_t a = 0; a < n_acct; a++)
        an_issue_finish_acct(a, na, touched.data(), balances, pendings, flags, present.data(), fin.data(), enc.data(), new_balances,
                             new_pendings, new_flags);
    return bad ? (long long)~bad : -1;
}
}
