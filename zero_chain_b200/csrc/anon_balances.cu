// Anonymous-transfer state updates of one block on the device (anon_balances.cuh): zk_balances_anonymous_block,
// zk_anonymous_calls_block (the same block with issue calls among the transfers) and their _device forms, all through one
// run_block; a block without issues takes the transfer-only passes.  One pass per stage, each one function per item and thread, all on the context's stream; the radix sort
// and the segmented scan are balances.cu's (zk_bal_sort, zk_bal_scan), and the workspace is the confidential call's
// buffer of the context.  The _device form only enqueues: a touched account that fails to read is left in an error word
// of the context, which the host form (and zk_ctx_sync after the _device form) reads back.
//
// Like balances.cu, the translation unit holds only Fr arithmetic and is compiled with everything inlined (ZK_HOT).
#define ZK_HOT 1
#include "internal.h"
#include "anon_balances.cuh"

using namespace zkbal;

constexpr int BT = 128;                 // threads per block

// one item per thread (a grid-stride loop would keep its counter live across the point arithmetic, and ptxas spills it)
#define BAL_FOR(i, n) for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i = (n))

static __global__ void __launch_bounds__(BT) k_an_touch(size_t n_tx, uint32_t n_acct, const uint32_t *__restrict__ members,
                                                        uint8_t *touched) {
    BAL_FOR(k, n_tx) an_touch(k, n_acct, members, touched);
}
// Point::read's square root and subgroup test: the register budget of k_bal_decode keeps it out of local memory
static __global__ void __maxnreg__(168) k_an_decode(size_t n, size_t n_tx, const uint8_t *__restrict__ kind, const uint8_t *__restrict__ tx_points,
                                                         const uint8_t *__restrict__ balances, const uint8_t *__restrict__ pendings,
                                                         const uint8_t *__restrict__ flags, const uint8_t *__restrict__ touched,
                                                         Ext *__restrict__ dec, uint8_t *__restrict__ ok) {
    BAL_FOR(p, n) an_decode(p, n_tx, tx_points, balances, pendings, flags, touched, dec, ok, kind);
}
static __global__ void __launch_bounds__(BT) k_an_tx(size_t n_tx, uint32_t n_acct, const uint32_t *__restrict__ members,
                                                     const uint8_t *__restrict__ applied, const Ext *__restrict__ dec,
                                                     const uint8_t *__restrict__ ok, uint32_t *__restrict__ keys, Pair *__restrict__ delta,
                                                     uint8_t *__restrict__ status, uint8_t *recv_any) {
    BAL_FOR(k, n_tx) an_tx(k, n_acct, members, applied, dec, ok, keys, delta, status, recv_any);
}
static __global__ void __launch_bounds__(BT) k_an_account(size_t n_acct, const uint8_t *__restrict__ flags, const uint8_t *__restrict__ touched,
                                                          const Ext *__restrict__ dec, const uint8_t *__restrict__ ok, Pair *__restrict__ roll_b,
                                                          Pair *__restrict__ roll_p, uint8_t *__restrict__ rflags, uint32_t *bad) {
    BAL_FOR(a, n_acct) bal_account(a, 0, flags, touched, dec, ok, roll_b, roll_p, rflags, bad);
}
static __global__ void __launch_bounds__(BT) k_an_totals(size_t n, uint32_t n_acct, const uint32_t *__restrict__ keys,
                                                         const uint32_t *__restrict__ vals, const Pair *__restrict__ excl,
                                                         const Pair *__restrict__ delta, Pair *__restrict__ tot, uint8_t *__restrict__ has) {
    BAL_FOR(j, n) an_totals(j, n, n_acct, keys, vals, excl, delta, tot, has);
}
static __global__ void __launch_bounds__(BT) k_an_acct_points(size_t n_acct, const uint8_t *__restrict__ touched,
                                                              const Pair *__restrict__ roll_b, const Pair *__restrict__ roll_p,
                                                              const uint8_t *__restrict__ rflags, const Pair *__restrict__ tot,
                                                              const uint8_t *__restrict__ has, const uint8_t *__restrict__ recv_any,
                                                              Ext *__restrict__ pts, uint8_t *__restrict__ present) {
    BAL_FOR(a, n_acct) bal_acct_points(a, 0, (uint32_t)n_acct, touched, roll_b, roll_p, rflags, tot, has, recv_any, pts, present);
}
static __global__ void __launch_bounds__(BT) k_an_encode(size_t n, const Ext *__restrict__ pts, Fr *__restrict__ prefix, uint32_t *__restrict__ enc) {
    BAL_FOR(c, (n + BAL_ENC_CHUNK - 1) / BAL_ENC_CHUNK) bal_encode_chunk(c, n, pts, prefix, enc);
}
static __global__ void __launch_bounds__(BT) k_an_finish_tx(size_t n, const uint32_t *__restrict__ members, const uint8_t *__restrict__ status,
                                                            const uint8_t *__restrict__ kind, const uint32_t *__restrict__ rd,
                                                            const uint8_t *__restrict__ enc_keys, const uint8_t *__restrict__ tx_points,
                                                            const uint8_t *__restrict__ tx_extra, const uint8_t *__restrict__ g_epoch,
                                                            const uint32_t *__restrict__ acct_enc, uint8_t *__restrict__ enc_balances,
                                                            uint8_t *__restrict__ verify_points) {
    BAL_FOR(s, n) an_finish_slot(s, members, status, enc_keys, tx_points, tx_extra, g_epoch, acct_enc, enc_balances, verify_points, kind, rd);
}
static __global__ void __launch_bounds__(BT) k_an_finish_acct(size_t n_acct, const uint8_t *__restrict__ touched,
                                                              const uint8_t *__restrict__ balances, const uint8_t *__restrict__ pendings,
                                                              const uint8_t *__restrict__ flags, const uint8_t *__restrict__ present,
                                                              const uint32_t *__restrict__ enc, uint8_t *__restrict__ new_balances,
                                                              uint8_t *__restrict__ new_pendings, uint8_t *__restrict__ new_flags) {
    BAL_FOR(a, n_acct) bal_finish_acct(a, 0, touched, balances, pendings, flags, present, enc, new_balances, new_pendings, new_flags);
}
// issue (zk_anonymous_calls_block only)
static __global__ void __launch_bounds__(BT) k_an_call_touch(size_t n_tx, uint32_t n_acct, const uint8_t *__restrict__ kind,
                                                             const uint32_t *__restrict__ members, uint8_t *touched, uint32_t *first) {
    BAL_FOR(k, n_tx) an_call_touch(k, n_acct, kind, members, touched, first);
}
static __global__ void __launch_bounds__(BT) k_an_call_tx(size_t n_tx, uint32_t n_acct, const uint8_t *__restrict__ kind,
                                                          const uint32_t *__restrict__ members, const uint8_t *__restrict__ applied,
                                                          const Ext *__restrict__ dec, const uint8_t *__restrict__ ok, uint32_t *__restrict__ keys,
                                                          Pair *__restrict__ delta, uint8_t *__restrict__ status, uint8_t *recv_any,
                                                          uint32_t *__restrict__ ikeys, Ext *__restrict__ ipts) {
    BAL_FOR(k, n_tx) an_call_tx(k, n_acct, kind, members, applied, dec, ok, keys, delta, status, recv_any, ikeys, ipts);
}
static __global__ void __launch_bounds__(BT) k_an_issue_account(size_t n_acct, size_t n_tx, const uint8_t *__restrict__ flags,
                                                                const uint8_t *__restrict__ touched, const uint32_t *__restrict__ first,
                                                                const uint32_t *__restrict__ ikeys, const uint32_t *__restrict__ ivals,
                                                                const Ext *__restrict__ dec, const uint8_t *__restrict__ ok,
                                                                Pair *__restrict__ roll_b, Pair *__restrict__ roll_p, uint8_t *__restrict__ rflags,
                                                                uint32_t *__restrict__ fin, uint32_t *bad) {
    BAL_FOR(a, n_acct) an_issue_account(a, n_tx, flags, touched, first, ikeys, ivals, dec, ok, roll_b, roll_p, rflags, fin, bad);
}
static __global__ void __launch_bounds__(BT) k_an_issue_read(size_t n, uint32_t n_acct, size_t n_tx, const uint8_t *__restrict__ kind,
                                                             const uint8_t *__restrict__ status, const uint32_t *__restrict__ members,
                                                             const uint32_t *__restrict__ first, const uint32_t *__restrict__ ikeys,
                                                             const uint32_t *__restrict__ ivals, uint32_t *__restrict__ rd) {
    BAL_FOR(e, n) an_issue_read(e, n_acct, n_tx, kind, status, members, first, ikeys, ivals, rd);
}
static __global__ void __launch_bounds__(BT) k_an_issued(size_t n_tx, uint32_t n_acct, const uint8_t *__restrict__ kind,
                                                         const uint8_t *__restrict__ status, const uint32_t *__restrict__ enc,
                                                         uint8_t *__restrict__ issued) {
    BAL_FOR(k, n_tx) an_issued(k, n_acct, kind, status, enc, issued);
}
static __global__ void __launch_bounds__(BT) k_an_issue_finish_acct(size_t n_acct, const uint8_t *__restrict__ touched,
                                                                    const uint8_t *__restrict__ balances, const uint8_t *__restrict__ pendings,
                                                                    const uint8_t *__restrict__ flags, const uint8_t *__restrict__ present,
                                                                    const uint32_t *__restrict__ fin, const uint32_t *__restrict__ enc,
                                                                    uint8_t *__restrict__ new_balances, uint8_t *__restrict__ new_pendings,
                                                                    uint8_t *__restrict__ new_flags) {
    BAL_FOR(a, n_acct) an_issue_finish_acct(a, (uint32_t)n_acct, touched, balances, pendings, flags, present, fin, enc, new_balances,
                                            new_pendings, new_flags);
}

struct AnonWork {
    uint32_t *keys0, *keys1, *vals0, *vals1, *hist, *totals;
    uint8_t *touched, *recv_any, *rflags, *present, *ok, *has, *head;
    Ext *dec, *pts;
    Pair *delta, *roll_b, *roll_p, *tot, *excl;
    Fr *prefix;
    uint32_t *enc;
    std::vector<size_t> lvl_n;                // items per scan level
    std::vector<Pair *> lvl_agg, lvl_out;     // level l >= 1: the aggregates and the scan of level l
    std::vector<uint8_t *> lvl_head;
    // issues: the first transfer touch of each account, the issue sort, the final balance's issue, each entry's read
    uint32_t *first, *ikeys0, *ikeys1, *ivals0, *ivals1, *fin, *rd;
};

// the counter-scan totals of zk_bal_sort: at most this many (balances.cu's SCAN_SEGMENTS)
constexpr size_t SORT_TOTALS = 1024;

// points to encode: each account's rolled balance and final pending, then each transaction's issue pair when calls
static size_t n_points(size_t n_tx, size_t n_acct, bool calls) { return 4 * n_acct + (calls ? 2 * n_tx : 0); }

static size_t carve(Carve &c, AnonWork &w, size_t n_tx, size_t n_acct, bool calls) {
    const size_t ne = AN_RING * n_tx, nd = AN_TX_POINTS * n_tx + 4 * n_acct, np = n_points(n_tx, n_acct, calls);
    const size_t n_tiles = (ne + BAL_SORT_TILE - 1) / BAL_SORT_TILE;
    w.keys0 = c.take<uint32_t>(ne); w.keys1 = c.take<uint32_t>(ne); w.vals0 = c.take<uint32_t>(ne); w.vals1 = c.take<uint32_t>(ne);
    w.hist = c.take<uint32_t>(BAL_RADIX * n_tiles); w.totals = c.take<uint32_t>(SORT_TOTALS);
    // touched and recv_any are next to each other: one memset clears both
    w.touched = c.take<uint8_t>(2 * n_acct); w.recv_any = w.touched ? w.touched + n_acct : nullptr;
    w.rflags = c.take<uint8_t>(n_acct); w.present = c.take<uint8_t>(n_acct); w.ok = c.take<uint8_t>(nd);
    w.has = c.take<uint8_t>(2 * n_acct); w.head = c.take<uint8_t>(ne);
    w.dec = c.take<Ext>(nd); w.pts = c.take<Ext>(np);
    w.delta = c.take<Pair>(ne); w.roll_b = c.take<Pair>(n_acct); w.roll_p = c.take<Pair>(n_acct); w.tot = c.take<Pair>(2 * n_acct);
    w.excl = c.take<Pair>(ne);
    w.prefix = c.take<Fr>(np); w.enc = c.take<uint32_t>(8 * np);
    w.lvl_n.assign(1, ne); w.lvl_agg.assign(1, nullptr); w.lvl_out.assign(1, w.excl); w.lvl_head.assign(1, w.head);
    for (size_t n = ne; n > BAL_SCAN_CHUNK;) {
        n = (n + BAL_SCAN_CHUNK - 1) / BAL_SCAN_CHUNK;
        w.lvl_n.push_back(n);
        w.lvl_agg.push_back(c.take<Pair>(n));
        w.lvl_out.push_back(c.take<Pair>(n));
        w.lvl_head.push_back(c.take<uint8_t>(n));
    }
    const size_t ni = calls ? n_tx : 0, na = calls ? n_acct : 0;
    w.first = c.take<uint32_t>(na); w.fin = c.take<uint32_t>(na); w.rd = c.take<uint32_t>(calls ? ne : 0);
    w.ikeys0 = c.take<uint32_t>(ni); w.ikeys1 = c.take<uint32_t>(ni); w.ivals0 = c.take<uint32_t>(ni); w.ivals1 = c.take<uint32_t>(ni);
    return c.off;
}

static unsigned grid(size_t n) { return (unsigned)(n ? (n + BT - 1) / BT : 1); }

// kind NULL: every transaction is an anonymous transfer (zk_balances_anonymous_block), and issued is not written
static int run_block(zk_ctx *ctx, size_t n_acct, const uint8_t *keys, const uint8_t *balances, const uint8_t *pendings, const uint8_t *acct_flags,
                     size_t n_tx, const uint8_t *kind, const uint32_t *members, const uint8_t *tx_points, const uint8_t *tx_extra,
                     const uint8_t *g_epoch, const uint8_t *applied, uint8_t *enc_balances, uint8_t *verify_points, uint8_t *issued,
                     uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags, DevBuf &buf) {
    cudaStream_t st = ctx->stream;
    const bool calls = kind && n_tx;
    if (!calls) kind = nullptr;
    AnonWork w;
    Carve sizing;
    ZK_TRY(buf.reserve(carve(sizing, w, n_tx, n_acct, calls)));
    Carve c;
    c.base = buf.as<uint8_t>();
    carve(c, w, n_tx, n_acct, calls);
    const size_t ne = AN_RING * n_tx, nd = AN_TX_POINTS * n_tx + 4 * n_acct, np = n_points(n_tx, n_acct, calls), ntp = AN_TX_POINTS * n_tx;
    const uint32_t na = (uint32_t)n_acct;

    ZK_CUDA(cudaMemsetAsync(w.touched, 0, 2 * n_acct, st));
    ZK_CUDA(cudaMemsetAsync(w.has, 0, 2 * n_acct, st));
    // the failing-account word: an error word of the context, reported (and cleared) by zk_check_err_flag
    uint32_t *bad = reinterpret_cast<uint32_t *>(ctx->d_err + ZK_ERR_SLOT_ACCOUNT);
    const uint32_t *iskeys = nullptr, *isvals = nullptr;
    if (calls) {
        ZK_CUDA(cudaMemsetAsync(w.first, 0xFF, sizeof(uint32_t) * n_acct, st));
        k_an_call_touch<<<grid(n_tx), BT, 0, st>>>(n_tx, na, kind, members, w.touched, w.first);
        k_an_decode<<<grid(nd), BT, 0, st>>>(nd, n_tx, kind, tx_points, balances, pendings, acct_flags, w.touched, w.dec, w.ok);
        k_an_call_tx<<<grid(n_tx), BT, 0, st>>>(n_tx, na, kind, members, applied, w.dec, w.ok, w.keys0, w.delta, tx_status, w.recv_any,
                                                w.ikeys0, w.pts + 4 * n_acct);
        ZK_CUDA(cudaGetLastError());
        // the applied issues grouped by issuer, in block order inside an issuer
        ZK_TRY(zk_bal_sort(ctx, n_tx, n_acct, w.ikeys0, w.ikeys1, w.ivals0, w.ivals1, w.hist, w.totals, &iskeys, &isvals));
        k_an_issue_account<<<grid(n_acct), BT, 0, st>>>(n_acct, n_tx, acct_flags, w.touched, w.first, iskeys, isvals, w.dec, w.ok, w.roll_b,
                                                        w.roll_p, w.rflags, w.fin, bad);
    } else {
        if (n_tx) k_an_touch<<<grid(n_tx), BT, 0, st>>>(n_tx, na, members, w.touched);
        k_an_decode<<<grid(nd), BT, 0, st>>>(nd, n_tx, nullptr, tx_points, balances, pendings, acct_flags, w.touched, w.dec, w.ok);
        if (n_tx) k_an_tx<<<grid(n_tx), BT, 0, st>>>(n_tx, na, members, applied, w.dec, w.ok, w.keys0, w.delta, tx_status, w.recv_any);
        k_an_account<<<grid(n_acct), BT, 0, st>>>(n_acct, acct_flags, w.touched, w.dec + ntp, w.ok + ntp, w.roll_b, w.roll_p, w.rflags, bad);
    }
    ZK_CUDA(cudaGetLastError());
    if (n_tx) {
        // the entries grouped by key; each key's total is its last element's exclusive sum plus its own delta
        const uint32_t *skeys, *svals;
        ZK_TRY(zk_bal_sort(ctx, ne, n_acct, w.keys0, w.keys1, w.vals0, w.vals1, w.hist, w.totals, &skeys, &svals));
        ZK_TRY(zk_bal_scan(ctx, skeys, svals, w.delta, w.lvl_n.size(), w.lvl_n.data(), w.lvl_agg.data(), w.lvl_out.data(), w.lvl_head.data()));
        k_an_totals<<<grid(ne), BT, 0, st>>>(ne, na, skeys, svals, w.excl, w.delta, w.tot, w.has);
        ZK_CUDA(cudaGetLastError());
    }
    k_an_acct_points<<<grid(n_acct), BT, 0, st>>>(n_acct, w.touched, w.roll_b, w.roll_p, w.rflags, w.tot, w.has, w.recv_any, w.pts, w.present);
    if (calls)
        k_an_issue_read<<<grid(ne), BT, 0, st>>>(ne, na, n_tx, kind, tx_status, members, w.first, iskeys, isvals, w.rd);
    k_an_encode<<<grid((np + BAL_ENC_CHUNK - 1) / BAL_ENC_CHUNK), BT, 0, st>>>(np, w.pts, w.prefix, w.enc);
    if (n_tx)
        k_an_finish_tx<<<grid(AN_VERIFY_POINTS * n_tx), BT, 0, st>>>(AN_VERIFY_POINTS * n_tx, members, tx_status, kind, calls ? w.rd : nullptr,
                                                                     keys, tx_points, tx_extra, g_epoch, w.enc, enc_balances, verify_points);
    if (calls) {
        k_an_issued<<<grid(n_tx), BT, 0, st>>>(n_tx, na, kind, tx_status, w.enc, issued);
        k_an_issue_finish_acct<<<grid(n_acct), BT, 0, st>>>(n_acct, w.touched, balances, pendings, acct_flags, w.present, w.fin, w.enc,
                                                            new_balances, new_pendings, new_flags);
    } else {
        k_an_finish_acct<<<grid(n_acct), BT, 0, st>>>(n_acct, w.touched, balances, pendings, acct_flags, w.present, w.enc, new_balances,
                                                      new_pendings, new_flags);
    }
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

// kind / issued: checked when calls (zk_anonymous_calls_block)
static int check_args(const char *fn, zk_ctx *ctx, size_t n_accounts, const void *keys, const void *balances, const void *pendings,
                      const void *acct_flags, size_t n_tx, bool calls, const void *kind, const void *members, const void *tx_points,
                      const void *tx_extra, const void *g_epoch, const void *applied, const void *enc_balances, const void *verify_points,
                      const void *issued, const void *tx_status, const void *new_balances, const void *new_pendings, const void *new_flags) {
    if (!ctx || (n_accounts && (!keys || !balances || !pendings || !acct_flags || !new_balances || !new_pendings || !new_flags)) ||
        (n_tx && (!members || !tx_points || !tx_extra || !g_epoch || !applied || !enc_balances || !verify_points || !tx_status)) ||
        (n_tx && calls && (!kind || !issued))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (n_accounts > BAL_MAX || n_tx > AN_MAX_TX) {
        zk_set_error("%s: n_accounts = %zu, n_tx = %zu: at most %u accounts and %u transactions", fn, n_accounts, n_tx, BAL_MAX, AN_MAX_TX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

// the host forms; kind NULL: no issue in the block
static int host_block(zk_ctx *ctx, size_t n_accounts, const uint8_t *keys, const uint8_t *balances, const uint8_t *pendings,
                      const uint8_t *acct_flags, size_t n_tx, const uint8_t *kind, const uint32_t *members, const uint8_t *tx_points,
                      const uint8_t *tx_extra, const uint8_t *g_epoch, const uint8_t *applied, uint8_t *enc_balances, uint8_t *verify_points,
                      uint8_t *issued, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags) {
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const size_t nk = kind ? n_tx : 0;
    const uint8_t *ky, *b, *p, *f, *kd, *tp, *tx, *ge, *ap;
    const uint32_t *m;
    uint8_t *eb, *vpt, *is, *ts, *nb, *npd, *nf;
    Stage io;
    io.in(keys, ky, 32 * n_accounts); io.in(balances, b, 64 * n_accounts); io.in(pendings, p, 64 * n_accounts);
    io.in(acct_flags, f, n_accounts);
    io.in(kind, kd, nk); io.in(members, m, AN_RING * n_tx); io.in(tx_points, tp, 32 * AN_TX_POINTS * n_tx); io.in(tx_extra, tx, 64 * n_tx);
    io.in(g_epoch, ge, n_tx ? 32 : 0); io.in(applied, ap, n_tx);
    io.out(enc_balances, eb, 64 * (size_t)AN_RING * n_tx); io.out(verify_points, vpt, 32 * (size_t)AN_VERIFY_POINTS * n_tx);
    io.inout(issued, is, 64 * nk);                // the entries no applied issue writes keep the caller's bytes
    io.out(tx_status, ts, n_tx);
    io.out(new_balances, nb, 64 * n_accounts); io.out(new_pendings, npd, 64 * n_accounts); io.out(new_flags, nf, n_accounts);
    ZK_TRY(io.up(ctx));
    ZK_TRY(run_block(ctx, n_accounts, ky, b, p, f, n_tx, kd, m, tp, tx, ge, ap, eb, vpt, is, ts, nb, npd, nf, ctx->bal));
    ZK_TRY(io.down(ctx));
    return zk_check_err_flag(ctx);     // synchronises the stream; ZK_ERR_DECODE names a touched account that failed to read
}

extern "C" int zk_balances_anonymous_block_device(zk_ctx *ctx, size_t n_accounts, const uint8_t *d_keys, const uint8_t *d_balances,
                                                  const uint8_t *d_pendings, const uint8_t *d_acct_flags, size_t n_tx, const uint32_t *d_members,
                                                  const uint8_t *d_tx_points, const uint8_t *d_tx_extra, const uint8_t *d_g_epoch,
                                                  const uint8_t *d_applied, uint8_t *d_enc_balances, uint8_t *d_verify_points,
                                                  uint8_t *d_tx_status, uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags) {
    ZK_TRY(check_args("zk_balances_anonymous_block_device", ctx, n_accounts, d_keys, d_balances, d_pendings, d_acct_flags, n_tx, false,
                      nullptr, d_members, d_tx_points, d_tx_extra, d_g_epoch, d_applied, d_enc_balances, d_verify_points, nullptr,
                      d_tx_status, d_new_balances, d_new_pendings, d_new_flags));
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return run_block(ctx, n_accounts, d_keys, d_balances, d_pendings, d_acct_flags, n_tx, nullptr, d_members, d_tx_points, d_tx_extra,
                     d_g_epoch, d_applied, d_enc_balances, d_verify_points, nullptr, d_tx_status, d_new_balances, d_new_pendings,
                     d_new_flags, ctx->bal);
}

extern "C" int zk_balances_anonymous_block(zk_ctx *ctx, size_t n_accounts, const uint8_t *keys, const uint8_t *balances, const uint8_t *pendings,
                                           const uint8_t *acct_flags, size_t n_tx, const uint32_t *members, const uint8_t *tx_points,
                                           const uint8_t *tx_extra, const uint8_t *g_epoch, const uint8_t *applied, uint8_t *enc_balances,
                                           uint8_t *verify_points, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings,
                                           uint8_t *new_flags) {
    ZK_TRY(check_args("zk_balances_anonymous_block", ctx, n_accounts, keys, balances, pendings, acct_flags, n_tx, false, nullptr, members,
                      tx_points, tx_extra, g_epoch, applied, enc_balances, verify_points, nullptr, tx_status, new_balances, new_pendings,
                      new_flags));
    return host_block(ctx, n_accounts, keys, balances, pendings, acct_flags, n_tx, nullptr, members, tx_points, tx_extra, g_epoch, applied,
                      enc_balances, verify_points, nullptr, tx_status, new_balances, new_pendings, new_flags);
}

extern "C" int zk_anonymous_calls_block_device(zk_ctx *ctx, size_t n_accounts, const uint8_t *d_keys, const uint8_t *d_balances,
                                               const uint8_t *d_pendings, const uint8_t *d_acct_flags, size_t n_tx, const uint8_t *d_kind,
                                               const uint32_t *d_members, const uint8_t *d_tx_points, const uint8_t *d_tx_extra,
                                               const uint8_t *d_g_epoch, const uint8_t *d_applied, uint8_t *d_enc_balances,
                                               uint8_t *d_verify_points, uint8_t *d_issued, uint8_t *d_tx_status, uint8_t *d_new_balances,
                                               uint8_t *d_new_pendings, uint8_t *d_new_flags) {
    ZK_TRY(check_args("zk_anonymous_calls_block_device", ctx, n_accounts, d_keys, d_balances, d_pendings, d_acct_flags, n_tx, true, d_kind,
                      d_members, d_tx_points, d_tx_extra, d_g_epoch, d_applied, d_enc_balances, d_verify_points, d_issued, d_tx_status,
                      d_new_balances, d_new_pendings, d_new_flags));
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return run_block(ctx, n_accounts, d_keys, d_balances, d_pendings, d_acct_flags, n_tx, d_kind, d_members, d_tx_points, d_tx_extra,
                     d_g_epoch, d_applied, d_enc_balances, d_verify_points, d_issued, d_tx_status, d_new_balances, d_new_pendings,
                     d_new_flags, ctx->bal);
}

extern "C" int zk_anonymous_calls_block(zk_ctx *ctx, size_t n_accounts, const uint8_t *keys, const uint8_t *balances, const uint8_t *pendings,
                                        const uint8_t *acct_flags, size_t n_tx, const uint8_t *kind, const uint32_t *members,
                                        const uint8_t *tx_points, const uint8_t *tx_extra, const uint8_t *g_epoch, const uint8_t *applied,
                                        uint8_t *enc_balances, uint8_t *verify_points, uint8_t *issued, uint8_t *tx_status,
                                        uint8_t *new_balances, uint8_t *new_pendings, uint8_t *new_flags) {
    ZK_TRY(check_args("zk_anonymous_calls_block", ctx, n_accounts, keys, balances, pendings, acct_flags, n_tx, true, kind, members, tx_points,
                      tx_extra, g_epoch, applied, enc_balances, verify_points, issued, tx_status, new_balances, new_pendings, new_flags));
    // a block of transfers only takes zk_balances_anonymous_block's passes
    bool other = false;
    for (size_t k = 0; k < n_tx && !other; k++) other = kind[k] != AN_TRANSFER;
    return host_block(ctx, n_accounts, keys, balances, pendings, acct_flags, n_tx, other ? kind : nullptr, members, tx_points, tx_extra,
                      g_epoch, applied, enc_balances, verify_points, issued, tx_status, new_balances, new_pendings, new_flags);
}
