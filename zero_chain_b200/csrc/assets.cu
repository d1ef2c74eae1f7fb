// Encrypted-asset calls of one block on the device (assets.cuh): zk_assets_block and its _device form.  One pass per
// stage, each one function per item and thread, all on the context's stream; the radix sort, the counter prefix sum and
// the segmented scan are balances.cu's (zk_bal_sort, zk_bal_prefix_sum, zk_bal_scan), and the workspace is the
// confidential call's buffer of the context.  The _device form only enqueues: a touched slot that fails to read is left
// in an error word of the context, which the host form (and zk_ctx_sync after the _device form) reads back.
//
// Like balances.cu, the translation unit holds only Fr arithmetic and is compiled with everything inlined (ZK_HOT).
#define ZK_HOT 1
#include "internal.h"
#include "assets.cuh"

using namespace zkbal;

constexpr int BT = 128;                 // threads per block
constexpr size_t SORT_TOTALS = 1024;    // the counter-scan totals of zk_bal_sort / zk_bal_prefix_sum (balances.cu's SCAN_SEGMENTS)

// one item per thread (a grid-stride loop would keep its counter live across the point arithmetic, and ptxas spills it)
#define BAL_FOR(i, n) for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i = (n))

static __global__ void __launch_bounds__(BT) k_as_touch(size_t n_tx, uint32_t n, const uint8_t *__restrict__ kind,
                                                        const uint32_t *__restrict__ slot_a, const uint32_t *__restrict__ slot_b,
                                                        uint8_t *touched, uint32_t *first) {
    BAL_FOR(k, n_tx) as_touch(k, n, kind, slot_a, slot_b, touched, first);
}
// Point::read's square root and subgroup test: the register budget of k_bal_decode keeps it out of local memory
static __global__ void __maxnreg__(168) k_as_decode(size_t np, size_t n_tx, const uint8_t *__restrict__ tx_points,
                                                         const uint8_t *__restrict__ balances, const uint8_t *__restrict__ pendings,
                                                         const uint8_t *__restrict__ flags, const uint8_t *__restrict__ touched,
                                                         Ext *__restrict__ dec, uint8_t *__restrict__ ok) {
    BAL_FOR(p, np) bal_decode(p, n_tx, tx_points, balances, pendings, flags, touched, dec, ok);
}
static __global__ void __launch_bounds__(BT) k_as_tx(size_t n_tx, uint32_t n, const uint8_t *__restrict__ kind,
                                                     const uint32_t *__restrict__ slot_a, const uint32_t *__restrict__ slot_b,
                                                     const uint8_t *__restrict__ applied, const uint8_t *__restrict__ flags,
                                                     const uint32_t *__restrict__ first, const Ext *__restrict__ dec,
                                                     const uint8_t *__restrict__ ok, uint32_t *__restrict__ keys, uint8_t *__restrict__ ebits,
                                                     Pair *__restrict__ delta, uint8_t *__restrict__ status) {
    BAL_FOR(k, n_tx) as_tx(k, n, kind, slot_a, slot_b, applied, flags, first, dec, ok, keys, ebits, delta, status);
}
static __global__ void __launch_bounds__(BT) k_as_slot(size_t n, size_t n_tx, const uint8_t *__restrict__ touched,
                                                       const Ext *__restrict__ dec, const uint8_t *__restrict__ ok, Pair *__restrict__ base,
                                                       uint32_t *bad) {
    BAL_FOR(a, n) as_slot(a, n_tx, (uint32_t)n, touched, dec, ok, base, bad);
}
static __global__ void __launch_bounds__(BT) k_as_pos(size_t ne, const uint32_t *__restrict__ skeys, const uint32_t *__restrict__ svals,
                                                      const uint8_t *__restrict__ ebits, uint32_t *__restrict__ pos, uint32_t *__restrict__ cnt) {
    BAL_FOR(j, ne) as_pos(j, skeys, svals, ebits, pos, cnt);
}
static __global__ void __launch_bounds__(BT) k_as_roll(size_t n, const uint32_t *__restrict__ skeys, const uint32_t *__restrict__ svals,
                                                       const uint8_t *__restrict__ ebits, const uint32_t *__restrict__ pos,
                                                       const Pair *__restrict__ base, Pair *delta) {
    BAL_FOR(i, n) as_roll(i, skeys, svals, ebits, pos, base, delta);
}
static __global__ void __launch_bounds__(BT) k_as_segkeys(size_t ne, const uint32_t *__restrict__ skeys, const uint32_t *__restrict__ svals,
                                                          const uint8_t *__restrict__ ebits, uint32_t *__restrict__ seg) {
    BAL_FOR(j, ne) as_segkeys(j, skeys, svals, ebits, seg);
}
static __global__ void __launch_bounds__(BT) k_as_seg(size_t ne, uint32_t n, const uint32_t *__restrict__ skeys, const uint32_t *__restrict__ svals,
                                                      const uint32_t *__restrict__ seg, const uint8_t *__restrict__ ebits,
                                                      const uint8_t *__restrict__ flags, uint8_t *__restrict__ seg_info, uint8_t *seg_recv,
                                                      uint32_t *__restrict__ last) {
    BAL_FOR(j, ne) as_seg(j, ne, n, skeys, svals, seg, ebits, flags, seg_info, seg_recv, last);
}
static __global__ void __maxnreg__(200) k_as_tx_points(size_t n_tx, uint32_t n, const uint8_t *__restrict__ kind,
                                                            const uint8_t *__restrict__ status, const uint32_t *__restrict__ skeys,
                                                            const uint32_t *__restrict__ svals, const uint32_t *__restrict__ pos,
                                                            const uint32_t *__restrict__ seg, const uint8_t *__restrict__ seg_info,
                                                            const uint8_t *__restrict__ seg_recv, const uint8_t *__restrict__ flags,
                                                            const Pair *__restrict__ base, const Pair *__restrict__ excl,
                                                            const Pair *__restrict__ delta, Ext *__restrict__ pts, uint8_t *__restrict__ evf) {
    BAL_FOR(k, n_tx) as_tx_points(k, n, kind, status, skeys, svals, pos, seg, seg_info, seg_recv, flags, base, excl, delta, pts, evf);
}
static __global__ void __maxnreg__(200) k_as_slot_points(size_t n, size_t n_tx, const uint8_t *__restrict__ touched,
                                                              const uint8_t *__restrict__ flags, const uint32_t *__restrict__ skeys,
                                                              const uint32_t *__restrict__ svals, const uint32_t *__restrict__ last,
                                                              const uint32_t *__restrict__ seg, const uint8_t *__restrict__ seg_info,
                                                              const uint8_t *__restrict__ seg_recv, const Pair *__restrict__ base,
                                                              const Pair *__restrict__ excl, const Pair *__restrict__ delta,
                                                              Ext *__restrict__ pts, uint8_t *__restrict__ present) {
    BAL_FOR(a, n) as_slot_points(a, n_tx, (uint32_t)n, touched, flags, skeys, svals, last, seg, seg_info, seg_recv, base, excl, delta, pts, present);
}
static __global__ void __launch_bounds__(BT) k_as_encode(size_t np, const Ext *__restrict__ pts, Fr *__restrict__ prefix, uint32_t *__restrict__ enc) {
    BAL_FOR(c, (np + BAL_ENC_CHUNK - 1) / BAL_ENC_CHUNK) bal_encode_chunk(c, np, pts, prefix, enc);
}
static __global__ void __launch_bounds__(BT) k_as_finish_tx(size_t n_tx, const uint8_t *__restrict__ kind, const uint8_t *__restrict__ status,
                                                            const uint8_t *__restrict__ evf, const uint32_t *__restrict__ enc,
                                                            uint8_t *__restrict__ balance_sender, uint8_t *__restrict__ balance_after,
                                                            uint8_t *__restrict__ event_ct, uint8_t *__restrict__ event_flags) {
    BAL_FOR(k, n_tx) as_finish_tx(k, kind, status, evf, enc, balance_sender, balance_after, event_ct, event_flags);
}
static __global__ void __launch_bounds__(BT) k_as_finish_slot(size_t n, size_t n_tx, const uint8_t *__restrict__ touched,
                                                              const uint32_t *__restrict__ first, const uint8_t *__restrict__ balances,
                                                              const uint8_t *__restrict__ pendings, const uint8_t *__restrict__ flags,
                                                              const uint8_t *__restrict__ present, const uint32_t *__restrict__ enc,
                                                              uint8_t *__restrict__ new_balances, uint8_t *__restrict__ new_pendings,
                                                              uint8_t *__restrict__ new_flags) {
    BAL_FOR(a, n) as_finish_slot(a, n_tx, touched, first, balances, pendings, flags, present, enc, new_balances, new_pendings, new_flags);
}

struct AssetWork {
    uint32_t *keys0, *keys1, *vals0, *vals1, *hist, *totals, *first, *pos, *seg, *last;
    uint8_t *touched, *present, *ok, *ebits, *seg_info, *seg_recv, *evf, *head;
    Ext *dec, *pts;
    Pair *delta, *base, *excl;
    Fr *prefix;
    uint32_t *enc;
    std::vector<size_t> lvl_n;                // items per scan level
    std::vector<Pair *> lvl_agg, lvl_out;     // level l >= 1: the aggregates and the scan of level l
    std::vector<uint8_t *> lvl_head;
};

static size_t carve(Carve &c, AssetWork &w, size_t n_tx, size_t n) {
    const size_t ne = AS_ELEMS * n_tx, np = 4 * n_tx + 4 * n, n_tiles = (ne + BAL_SORT_TILE - 1) / BAL_SORT_TILE;
    w.keys0 = c.take<uint32_t>(ne); w.keys1 = c.take<uint32_t>(ne); w.vals0 = c.take<uint32_t>(ne); w.vals1 = c.take<uint32_t>(ne);
    w.hist = c.take<uint32_t>(BAL_RADIX * n_tiles); w.totals = c.take<uint32_t>(SORT_TOTALS);
    w.first = c.take<uint32_t>(n); w.pos = c.take<uint32_t>(ne); w.seg = c.take<uint32_t>(ne); w.last = c.take<uint32_t>(2 * n);
    w.touched = c.take<uint8_t>(n); w.present = c.take<uint8_t>(n); w.ok = c.take<uint8_t>(np); w.ebits = c.take<uint8_t>(ne);
    w.seg_info = c.take<uint8_t>(ne); w.seg_recv = c.take<uint8_t>(ne); w.evf = c.take<uint8_t>(n_tx); w.head = c.take<uint8_t>(ne);
    w.dec = c.take<Ext>(np); w.pts = c.take<Ext>(np);
    w.delta = c.take<Pair>(ne); w.base = c.take<Pair>(2 * n); w.excl = c.take<Pair>(ne);
    w.prefix = c.take<Fr>(np); w.enc = c.take<uint32_t>(8 * np);
    w.lvl_n.assign(1, ne); w.lvl_agg.assign(1, nullptr); w.lvl_out.assign(1, w.excl); w.lvl_head.assign(1, w.head);
    for (size_t m = ne; m > BAL_SCAN_CHUNK;) {
        m = (m + BAL_SCAN_CHUNK - 1) / BAL_SCAN_CHUNK;
        w.lvl_n.push_back(m);
        w.lvl_agg.push_back(c.take<Pair>(m));
        w.lvl_out.push_back(c.take<Pair>(m));
        w.lvl_head.push_back(c.take<uint8_t>(m));
    }
    return c.off;
}

static unsigned grid(size_t n) { return (unsigned)(n ? (n + BT - 1) / BT : 1); }

static int run_block(zk_ctx *ctx, size_t n, const uint8_t *balances, const uint8_t *pendings, const uint8_t *slot_flags, size_t n_tx,
                     const uint8_t *kind, const uint32_t *slot_a, const uint32_t *slot_b, const uint8_t *tx_points, const uint8_t *applied,
                     uint8_t *balance_sender, uint8_t *balance_after, uint8_t *event_ct, uint8_t *event_flags, uint8_t *tx_status,
                     uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags, DevBuf &buf) {
    cudaStream_t st = ctx->stream;
    AssetWork w;
    Carve sizing;
    ZK_TRY(buf.reserve(carve(sizing, w, n_tx, n)));
    Carve c;
    c.base = buf.as<uint8_t>();
    carve(c, w, n_tx, n);
    const size_t ne = AS_ELEMS * n_tx, np = 4 * n_tx + 4 * n;
    const uint32_t n32 = (uint32_t)n;

    ZK_CUDA(cudaMemsetAsync(w.touched, 0, n, st));
    ZK_CUDA(cudaMemsetAsync(w.first, 0xFF, 4 * n, st));
    ZK_CUDA(cudaMemsetAsync(w.last, 0xFF, 8 * n, st));
    // the failing-slot word: an error word of the context, reported (and cleared) by zk_check_err_flag
    uint32_t *bad = reinterpret_cast<uint32_t *>(ctx->d_err + ZK_ERR_SLOT_ACCOUNT);
    if (n_tx) k_as_touch<<<grid(n_tx), BT, 0, st>>>(n_tx, n32, kind, slot_a, slot_b, w.touched, w.first);
    k_as_decode<<<grid(np), BT, 0, st>>>(np, n_tx, tx_points, balances, pendings, slot_flags, w.touched, w.dec, w.ok);
    if (n_tx)
        k_as_tx<<<grid(n_tx), BT, 0, st>>>(n_tx, n32, kind, slot_a, slot_b, applied, slot_flags, w.first, w.dec, w.ok, w.keys0, w.ebits,
                                           w.delta, tx_status);
    k_as_slot<<<grid(n), BT, 0, st>>>(n, n_tx, w.touched, w.dec, w.ok, w.base, bad);
    ZK_CUDA(cudaGetLastError());
    const uint32_t *skeys = nullptr, *svals = nullptr;
    if (n_tx) {
        ZK_TRY(zk_bal_sort(ctx, ne, n, w.keys0, w.keys1, w.vals0, w.vals1, w.hist, w.totals, &skeys, &svals));
        k_as_pos<<<grid(ne), BT, 0, st>>>(ne, skeys, svals, w.ebits, w.pos, w.seg);
        k_as_roll<<<grid(2 * n_tx), BT, 0, st>>>(2 * n_tx, skeys, svals, w.ebits, w.pos, w.base, w.delta);
        ZK_CUDA(cudaGetLastError());
        // segment numbers: the scan restarts at every key change and at every head
        ZK_TRY(zk_bal_prefix_sum(ctx, w.seg, ne, w.totals));
        k_as_segkeys<<<grid(ne), BT, 0, st>>>(ne, skeys, svals, w.ebits, w.seg);
        ZK_CUDA(cudaGetLastError());
        ZK_TRY(zk_bal_scan(ctx, w.seg, svals, w.delta, w.lvl_n.size(), w.lvl_n.data(), w.lvl_agg.data(), w.lvl_out.data(), w.lvl_head.data()));
        ZK_CUDA(cudaMemsetAsync(w.seg_recv, 0, ne, st));
        k_as_seg<<<grid(ne), BT, 0, st>>>(ne, n32, skeys, svals, w.seg, w.ebits, slot_flags, w.seg_info, w.seg_recv, w.last);
        k_as_tx_points<<<grid(n_tx), BT, 0, st>>>(n_tx, n32, kind, tx_status, skeys, svals, w.pos, w.seg, w.seg_info, w.seg_recv, slot_flags,
                                                  w.base, w.excl, w.delta, w.pts, w.evf);
        ZK_CUDA(cudaGetLastError());
    }
    k_as_slot_points<<<grid(n), BT, 0, st>>>(n, n_tx, w.touched, slot_flags, skeys, svals, w.last, w.seg, w.seg_info, w.seg_recv, w.base,
                                             w.excl, w.delta, w.pts, w.present);
    k_as_encode<<<grid((np + BAL_ENC_CHUNK - 1) / BAL_ENC_CHUNK), BT, 0, st>>>(np, w.pts, w.prefix, w.enc);
    if (n_tx)
        k_as_finish_tx<<<grid(n_tx), BT, 0, st>>>(n_tx, kind, tx_status, w.evf, w.enc, balance_sender, balance_after, event_ct, event_flags);
    k_as_finish_slot<<<grid(n), BT, 0, st>>>(n, n_tx, w.touched, w.first, balances, pendings, slot_flags, w.present, w.enc, new_balances,
                                             new_pendings, new_flags);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

static int check_args(const char *fn, zk_ctx *ctx, size_t n_slots, const void *balances, const void *pendings, const void *slot_flags,
                      size_t n_tx, const void *kind, const void *slot_a, const void *slot_b, const void *tx_points, const void *applied,
                      const void *balance_sender, const void *balance_after, const void *event_ct, const void *event_flags,
                      const void *tx_status, const void *new_balances, const void *new_pendings, const void *new_flags) {
    if (!ctx || (n_slots && (!balances || !pendings || !slot_flags || !new_balances || !new_pendings || !new_flags)) ||
        (n_tx && (!kind || !slot_a || !slot_b || !tx_points || !applied || !balance_sender || !balance_after || !event_ct || !event_flags ||
                  !tx_status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (n_slots > BAL_MAX || n_tx > AS_MAX_TX) {
        zk_set_error("%s: n_slots = %zu, n_tx = %zu: at most %u slots and %u transactions", fn, n_slots, n_tx, BAL_MAX, AS_MAX_TX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

extern "C" int zk_assets_block_device(zk_ctx *ctx, size_t n_slots, const uint8_t *d_balances, const uint8_t *d_pendings,
                                      const uint8_t *d_slot_flags, size_t n_tx, const uint8_t *d_kind, const uint32_t *d_slot_a,
                                      const uint32_t *d_slot_b, const uint8_t *d_tx_points, const uint8_t *d_applied,
                                      uint8_t *d_balance_sender, uint8_t *d_balance_after, uint8_t *d_event_ct, uint8_t *d_event_flags,
                                      uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags) {
    ZK_TRY(check_args("zk_assets_block_device", ctx, n_slots, d_balances, d_pendings, d_slot_flags, n_tx, d_kind, d_slot_a, d_slot_b,
                      d_tx_points, d_applied, d_balance_sender, d_balance_after, d_event_ct, d_event_flags, d_tx_status, d_new_balances,
                      d_new_pendings, d_new_flags));
    if (!n_slots && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return run_block(ctx, n_slots, d_balances, d_pendings, d_slot_flags, n_tx, d_kind, d_slot_a, d_slot_b, d_tx_points, d_applied,
                     d_balance_sender, d_balance_after, d_event_ct, d_event_flags, d_tx_status, d_new_balances, d_new_pendings, d_new_flags,
                     ctx->bal);
}

extern "C" int zk_assets_block(zk_ctx *ctx, size_t n_slots, const uint8_t *balances, const uint8_t *pendings, const uint8_t *slot_flags,
                               size_t n_tx, const uint8_t *kind, const uint32_t *slot_a, const uint32_t *slot_b, const uint8_t *tx_points,
                               const uint8_t *applied, uint8_t *balance_sender, uint8_t *balance_after, uint8_t *event_ct,
                               uint8_t *event_flags, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags) {
    ZK_TRY(check_args("zk_assets_block", ctx, n_slots, balances, pendings, slot_flags, n_tx, kind, slot_a, slot_b, tx_points, applied,
                      balance_sender, balance_after, event_ct, event_flags, tx_status, new_balances, new_pendings, new_flags));
    if (!n_slots && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *b, *p, *f, *kd, *tp, *ap;
    const uint32_t *sa, *sb;
    uint8_t *bs, *ba, *ev, *ef, *ts, *nb, *npd, *nf;
    Stage io;
    io.in(balances, b, 64 * n_slots); io.in(pendings, p, 64 * n_slots); io.in(slot_flags, f, n_slots);
    io.in(kind, kd, n_tx); io.in(slot_a, sa, n_tx); io.in(slot_b, sb, n_tx); io.in(tx_points, tp, 128 * n_tx); io.in(applied, ap, n_tx);
    io.out(balance_sender, bs, 64 * n_tx);
    // only some of these entries are written
    io.inout(balance_after, ba, 64 * n_tx); io.inout(event_ct, ev, 128 * n_tx); io.inout(event_flags, ef, n_tx);
    io.out(tx_status, ts, n_tx);
    io.out(new_balances, nb, 64 * n_slots); io.out(new_pendings, npd, 64 * n_slots); io.out(new_flags, nf, n_slots);
    ZK_TRY(io.up(ctx));
    ZK_TRY(run_block(ctx, n_slots, b, p, f, n_tx, kd, sa, sb, tp, ap, bs, ba, ev, ef, ts, nb, npd, nf, ctx->bal));
    ZK_TRY(io.down(ctx));
    return zk_check_err_flag(ctx);     // synchronises the stream; ZK_ERR_DECODE names a touched slot that failed to read
}
