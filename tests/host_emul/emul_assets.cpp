// CPU unit-test harness of the PRODUCT's encrypted-asset header (zero_chain_b200/csrc/assets.cuh) compiled with
// ZK_HOST_EMUL: every pass of assets.cu run as a loop over its items, in the same order of passes and with the same
// workspace layout, checked by tests/test_host_emul_assets.py against the oracles.  Test infrastructure only — never
// linked into libzkb200.so.
#define ZK_HOST_EMUL 1
#include "assets.cuh"
#include <string.h>
#include <vector>

using namespace zkbal;

extern "C" {
// zk_assets_block on host arrays; returns -1, or the lowest named slot that fails to decode
long long emu_as_block(size_t n, const uint8_t *balances, const uint8_t *pendings, const uint8_t *flags, size_t n_tx, const uint8_t *kind,
                       const uint32_t *slot_a, const uint32_t *slot_b, const uint8_t *tx_points, const uint8_t *applied,
                       uint8_t *balance_sender, uint8_t *balance_after, uint8_t *event_ct, uint8_t *event_flags, uint8_t *status,
                       uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags) {
    const size_t ne = AS_ELEMS * n_tx, np = 4 * n_tx + 4 * n, n_tiles = (ne + BAL_SORT_TILE - 1) / BAL_SORT_TILE;
    std::vector<uint32_t> keys0(ne + 1), keys1(ne + 1), vals0(ne + 1), vals1(ne + 1), hist(BAL_RADIX * n_tiles + 1), enc(8 * np + 8),
        first(n + 1, AS_NONE), pos(ne + 1), seg(ne + 1), last(2 * n + 1, AS_NONE);
    std::vector<uint8_t> touched(n + 1), present(n + 1), ok(np + 1), ebits(ne + 1), seg_info(ne + 1), seg_recv(ne + 1), evf(n_tx + 1);
    std::vector<Ext> dec(np + 1), pts(np + 1);
    std::vector<Pair> delta(ne + 1), base(2 * n + 1);
    std::vector<Fr> prefix(np + 1);
    uint32_t bad = 0;
    const uint32_t n32 = (uint32_t)n;
    // the transactions run in reverse where the device runs them concurrently: the order of the threads must not matter
    for (size_t k = n_tx; k-- > 0;) as_touch(k, n32, kind, slot_a, slot_b, touched.data(), first.data());
    for (size_t p = 0; p < np; p++) bal_decode(p, n_tx, tx_points, balances, pendings, flags, touched.data(), dec.data(), ok.data());
    for (size_t k = 0; k < n_tx; k++)
        as_tx(k, n32, kind, slot_a, slot_b, applied, flags, first.data(), dec.data(), ok.data(), keys0.data(), ebits.data(), delta.data(), status);
    for (size_t a = 0; a < n; a++) as_slot(a, n_tx, n32, touched.data(), dec.data(), ok.data(), base.data(), &bad);
    const uint32_t *skeys = nullptr, *svals = nullptr;
    std::vector<std::vector<Pair>> out(1);
    if (n_tx) {
        int bits = 0;
        while (bits < 32 && ((2 * (uint64_t)n) >> bits)) bits++;
        const int passes = bits <= BAL_RADIX_BITS ? 1 : (bits + BAL_RADIX_BITS - 1) / BAL_RADIX_BITS;
        uint32_t *kin = keys0.data(), *vin = nullptr, *kout = keys1.data(), *vout = vals1.data();
        for (int p = 0; p < passes; p++) {
            std::fill(hist.begin(), hist.end(), 0);
            for (size_t t = n_tiles; t-- > 0;) bal_radix_hist(t, ne, kin, BAL_RADIX_BITS * p, n_tiles, hist.data());
            uint32_t run = 0;
            for (size_t i = 0; i < BAL_RADIX * n_tiles; i++) { const uint32_t v = hist[i]; hist[i] = run; run += v; }
            for (size_t t = n_tiles; t-- > 0;) bal_radix_scatter(t, ne, kin, vin, BAL_RADIX_BITS * p, n_tiles, hist.data(), kout, vout);
            kin = kout; vin = vout;
            kout = kin == keys1.data() ? keys0.data() : keys1.data();
            vout = vin == vals1.data() ? vals0.data() : vals1.data();
        }
        skeys = kin; svals = vin;
        for (size_t j = 0; j < ne; j++) as_pos(j, skeys, svals, ebits.data(), pos.data(), seg.data());
        for (size_t i = 2 * n_tx; i-- > 0;) as_roll(i, skeys, svals, ebits.data(), pos.data(), base.data(), delta.data());
        uint32_t run = 0;
        for (size_t j = 0; j < ne; j++) { const uint32_t v = seg[j]; seg[j] = run; run += v; }
        for (size_t j = 0; j < ne; j++) as_segkeys(j, skeys, svals, ebits.data(), seg.data());
        // zk_bal_scan keyed by the segment numbers
        std::vector<uint8_t> head(ne + 1);
        for (size_t j = 0; j < ne; j++) bal_heads(j, seg.data(), head.data());
        std::vector<size_t> ln(1, ne);
        std::vector<std::vector<Pair>> agg(1);
        out[0].resize(ne + 1);
        std::vector<std::vector<uint8_t>> hd(1, head);
        for (size_t m = ne; m > BAL_SCAN_CHUNK;) {
            m = (m + BAL_SCAN_CHUNK - 1) / BAL_SCAN_CHUNK;
            ln.push_back(m); agg.emplace_back(m + 1); out.emplace_back(m + 1); hd.emplace_back(m + 1);
        }
        const size_t L = ln.size();
        for (size_t l = 0; l + 1 < L; l++)
            for (size_t c = 0; c < ln[l + 1]; c++)
                bal_scan_up(c, ln[l], l ? agg[l].data() : delta.data(), l ? nullptr : svals, hd[l].data(), agg[l + 1].data(), hd[l + 1].data());
        for (size_t l = L; l-- > 0;)
            for (size_t c = 0; c * BAL_SCAN_CHUNK < ln[l]; c++)
                bal_scan_down(c, ln[l], l ? agg[l].data() : delta.data(), l ? nullptr : svals, hd[l].data(),
                              l + 1 < L ? out[l + 1].data() : nullptr, l == 0, out[l].data());
        for (size_t j = ne; j-- > 0;) as_seg(j, ne, n32, skeys, svals, seg.data(), ebits.data(), flags, seg_info.data(), seg_recv.data(), last.data());
        for (size_t k = 0; k < n_tx; k++)
            as_tx_points(k, n32, kind, status, skeys, svals, pos.data(), seg.data(), seg_info.data(), seg_recv.data(), flags, base.data(),
                         out[0].data(), delta.data(), pts.data(), evf.data());
    }
    for (size_t a = 0; a < n; a++)
        as_slot_points(a, n_tx, n32, touched.data(), flags, skeys, svals, last.data(), seg.data(), seg_info.data(), seg_recv.data(), base.data(),
                       out[0].data(), delta.data(), pts.data(), present.data());
    for (size_t c = 0; c * BAL_ENC_CHUNK < np; c++) bal_encode_chunk(c, np, pts.data(), prefix.data(), enc.data());
    for (size_t k = 0; k < n_tx; k++) as_finish_tx(k, kind, status, evf.data(), enc.data(), balance_sender, balance_after, event_ct, event_flags);
    for (size_t a = 0; a < n; a++)
        as_finish_slot(a, n_tx, touched.data(), first.data(), balances, pendings, flags, present.data(), enc.data(), new_balances, new_pendings,
                       new_flags);
    return bad ? (long long)~bad : -1;
}
}
