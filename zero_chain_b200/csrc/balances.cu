// Confidential-transfer balance updates of one block on the device (balances.cuh): zk_balances_confidential_block and its
// _device form.  One pass per stage, each one balances.cuh function per item and thread, all on the context's stream; the
// workspace stays in the context.  The _device form only enqueues: a touched account that fails to read is left in an
// error word of the context, which the host form (and zk_ctx_sync after the _device form) reads back.  The radix sort and
// the segmented scan (zk_bal_sort, zk_bal_scan) also serve the anonymous-transfer block of anon_balances.cu.
//
// Like elgamal.cu, the translation unit holds only Fr arithmetic and is compiled with everything inlined (ZK_HOT).
#define ZK_HOT 1
#include "internal.h"
#include "balances.cuh"

using namespace zkbal;

constexpr int BT = 128;                 // threads per block
constexpr int SCAN_THREADS = 1024;      // threads of a block of the radix counters' prefix sum
constexpr size_t SCAN_SEGMENTS = 1024;  // at most this many blocks in it, each of at least SCAN_MIN_SEG counters
constexpr size_t SCAN_MIN_SEG = 8192;

// one item per thread (a grid-stride loop would keep its counter live across the point arithmetic, and ptxas spills it)
#define BAL_FOR(i, n) for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i = (n))

static __global__ void __launch_bounds__(BT) k_bal_touch(size_t n_tx, uint32_t n_acct, const uint32_t *__restrict__ sender,
                                                         const uint32_t *__restrict__ recipient, uint32_t *__restrict__ keys, uint8_t *touched) {
    BAL_FOR(k, n_tx) bal_touch(k, n_acct, sender, recipient, keys, touched);
}
// Point::read's square root and subgroup test, and the two-point outputs: left at the default budget, ptxas spills a few
// words of these two kernels to local memory; a fixed register budget keeps everything in registers.
static __global__ void __maxnreg__(168) k_bal_decode(size_t n, size_t n_tx, const uint8_t *__restrict__ tx_points,
                                                          const uint8_t *__restrict__ balances, const uint8_t *__restrict__ pendings,
                                                          const uint8_t *__restrict__ flags, const uint8_t *__restrict__ touched,
                                                          Ext *__restrict__ dec, uint8_t *__restrict__ ok) {
    BAL_FOR(p, n) bal_decode(p, n_tx, tx_points, balances, pendings, flags, touched, dec, ok);
}
static __global__ void __launch_bounds__(BT) k_bal_tx(size_t n_tx, uint32_t n_acct, const uint32_t *__restrict__ sender,
                                                      const uint32_t *__restrict__ recipient, const uint8_t *__restrict__ applied,
                                                      const Ext *__restrict__ dec, const uint8_t *__restrict__ ok, Pair *__restrict__ delta,
                                                      uint8_t *__restrict__ status, uint8_t *recv_any) {
    BAL_FOR(k, n_tx) bal_tx(k, n_acct, sender, recipient, applied, dec, ok, delta, status, recv_any);
}
static __global__ void __launch_bounds__(BT) k_bal_account(size_t n_acct, size_t n_tx, const uint8_t *__restrict__ flags,
                                                           const uint8_t *__restrict__ touched, const Ext *__restrict__ dec,
                                                           const uint8_t *__restrict__ ok, Pair *__restrict__ roll_b, Pair *__restrict__ roll_p,
                                                           uint8_t *__restrict__ rflags, uint32_t *bad) {
    BAL_FOR(a, n_acct) bal_account(a, n_tx, flags, touched, dec, ok, roll_b, roll_p, rflags, bad);
}
static __global__ void __launch_bounds__(BT) k_bal_radix_hist(size_t n, const uint32_t *__restrict__ keys, int shift, size_t n_tiles,
                                                              uint32_t *__restrict__ hist) {
    BAL_FOR(t, n_tiles) bal_radix_hist(t, n, keys, shift, n_tiles, hist);
}
static __global__ void __launch_bounds__(BT) k_bal_radix_scatter(size_t n, const uint32_t *__restrict__ keys_in, const uint32_t *__restrict__ vals_in,
                                                                 int shift, size_t n_tiles, uint32_t *__restrict__ cursor,
                                                                 uint32_t *__restrict__ keys_out, uint32_t *__restrict__ vals_out) {
    BAL_FOR(t, n_tiles) bal_radix_scatter(t, n, keys_in, vals_in, shift, n_tiles, cursor, keys_out, vals_out);
}
// Exclusive prefix sum of the radix counters ([digit][tile], 2^8 x ceil(2 n_tx / 64) of them) in three passes: the sum of
// each of up to SCAN_SEGMENTS segments, a scan of those sums, and a scan of each segment from its carry.  In the last two a
// block's threads each take a contiguous run of their segment and the block scans the run totals.
static __global__ void __launch_bounds__(SCAN_THREADS) k_bal_counter_sums(const uint32_t *__restrict__ c, size_t n, size_t seg,
                                                                          uint32_t *__restrict__ totals) {
    __shared__ uint32_t part[SCAN_THREADS];
    const size_t s0 = blockIdx.x * seg, s1 = s0 + seg < n ? s0 + seg : n;
    uint32_t s = 0;
    for (size_t i = s0 + threadIdx.x; i < s1; i += SCAN_THREADS) s += c[i];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int d = SCAN_THREADS / 2; d > 0; d >>= 1) {
        if (threadIdx.x < (unsigned)d) part[threadIdx.x] += part[threadIdx.x + d];
        __syncthreads();
    }
    if (!threadIdx.x) totals[blockIdx.x] = part[0];
}
// block b: counters [b seg, (b + 1) seg) in place, starting from carry[b] (NULL: 0)
static __global__ void __launch_bounds__(SCAN_THREADS) k_bal_counter_scan(uint32_t *c, size_t n, size_t seg, const uint32_t *carry) {
    __shared__ uint32_t part[SCAN_THREADS];
    const size_t s0 = blockIdx.x * seg < n ? blockIdx.x * seg : n, s1 = s0 + seg < n ? s0 + seg : n;
    const size_t per = (s1 - s0 + SCAN_THREADS - 1) / SCAN_THREADS;
    const size_t i0 = s0 + threadIdx.x * per < s1 ? s0 + threadIdx.x * per : s1, i1 = i0 + per < s1 ? i0 + per : s1;
    uint32_t s = 0;
    for (size_t i = i0; i < i1; i++) s += c[i];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int d = 1; d < SCAN_THREADS; d <<= 1) {       // Hillis-Steele inclusive scan of the run totals
        const uint32_t v = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = (carry ? carry[blockIdx.x] : 0) + part[threadIdx.x] - s;
    for (size_t i = i0; i < i1; i++) { const uint32_t v = c[i]; c[i] = run; run += v; }
}
static __global__ void __launch_bounds__(BT) k_bal_heads(size_t n, const uint32_t *__restrict__ keys, uint8_t *__restrict__ head) {
    BAL_FOR(j, n) bal_heads(j, keys, head);
}
static __global__ void __launch_bounds__(BT) k_bal_scan_up(size_t n, const Pair *__restrict__ v, const uint32_t *__restrict__ idx,
                                                           const uint8_t *__restrict__ head, Pair *__restrict__ agg, uint8_t *__restrict__ agg_head) {
    BAL_FOR(c, (n + BAL_SCAN_CHUNK - 1) / BAL_SCAN_CHUNK) bal_scan_up(c, n, v, idx, head, agg, agg_head);
}
static __global__ void __launch_bounds__(BT) k_bal_scan_down(size_t n, const Pair *__restrict__ v, const uint32_t *__restrict__ idx,
                                                             const uint8_t *__restrict__ head, const Pair *__restrict__ carry, bool elements,
                                                             Pair *__restrict__ out) {
    BAL_FOR(c, (n + BAL_SCAN_CHUNK - 1) / BAL_SCAN_CHUNK) bal_scan_down(c, n, v, idx, head, carry, elements, out);
}
static __global__ void __maxnreg__(200) k_bal_tx_points(size_t n, uint32_t n_acct, const uint32_t *__restrict__ keys,
                                                             const uint32_t *__restrict__ vals, const Pair *__restrict__ excl,
                                                             const Pair *__restrict__ delta, const Pair *__restrict__ roll_b,
                                                             const uint8_t *__restrict__ rflags, const uint8_t *__restrict__ status,
                                                             Ext *__restrict__ pts, Pair *__restrict__ tot, uint8_t *__restrict__ has) {
    BAL_FOR(j, n) bal_tx_points(j, n, n_acct, keys, vals, excl, delta, roll_b, rflags, status, pts, tot, has);
}
static __global__ void __launch_bounds__(BT) k_bal_acct_points(size_t n_acct, size_t n_tx, const uint8_t *__restrict__ touched,
                                                               const Pair *__restrict__ roll_b, const Pair *__restrict__ roll_p,
                                                               const uint8_t *__restrict__ rflags, const Pair *__restrict__ tot,
                                                               const uint8_t *__restrict__ has, const uint8_t *__restrict__ recv_any,
                                                               Ext *__restrict__ pts, uint8_t *__restrict__ present) {
    BAL_FOR(a, n_acct) bal_acct_points(a, n_tx, (uint32_t)n_acct, touched, roll_b, roll_p, rflags, tot, has, recv_any, pts, present);
}
static __global__ void __launch_bounds__(BT) k_bal_encode(size_t n, const Ext *__restrict__ pts, Fr *__restrict__ prefix, uint32_t *__restrict__ enc) {
    BAL_FOR(c, (n + BAL_ENC_CHUNK - 1) / BAL_ENC_CHUNK) bal_encode_chunk(c, n, pts, prefix, enc);
}
static __global__ void __launch_bounds__(BT) k_bal_finish_tx(size_t n_tx, const uint8_t *__restrict__ status, const uint32_t *__restrict__ enc,
                                                             uint8_t *__restrict__ balance_sender, uint8_t *__restrict__ balance_after) {
    BAL_FOR(k, n_tx) bal_finish_tx(k, status, enc, balance_sender, balance_after);
}
static __global__ void __launch_bounds__(BT) k_bal_finish_acct(size_t n_acct, size_t n_tx, const uint8_t *__restrict__ touched,
                                                               const uint8_t *__restrict__ balances, const uint8_t *__restrict__ pendings,
                                                               const uint8_t *__restrict__ flags, const uint8_t *__restrict__ present,
                                                               const uint32_t *__restrict__ enc, uint8_t *__restrict__ new_balances,
                                                               uint8_t *__restrict__ new_pendings, uint8_t *__restrict__ new_flags) {
    BAL_FOR(a, n_acct) bal_finish_acct(a, n_tx, touched, balances, pendings, flags, present, enc, new_balances, new_pendings, new_flags);
}

struct BalWork {
    uint32_t *keys0, *keys1, *vals0, *vals1, *hist, *totals;
    uint8_t *touched, *recv_any, *rflags, *present, *ok, *has, *head;
    Ext *dec, *pts;
    Pair *delta, *roll_b, *roll_p, *tot, *excl;
    Fr *prefix;
    uint32_t *enc;
    std::vector<size_t> lvl_n;                // items per scan level
    std::vector<Pair *> lvl_agg, lvl_out;     // level l >= 1: the aggregates and the scan of level l
    std::vector<uint8_t *> lvl_head;
};

static size_t carve(Carve &c, BalWork &w, size_t n_tx, size_t n_acct) {
    const size_t ne = 2 * n_tx, np = 4 * n_tx + 4 * n_acct, n_tiles = (ne + BAL_SORT_TILE - 1) / BAL_SORT_TILE;
    w.keys0 = c.take<uint32_t>(ne); w.keys1 = c.take<uint32_t>(ne); w.vals0 = c.take<uint32_t>(ne); w.vals1 = c.take<uint32_t>(ne);
    w.hist = c.take<uint32_t>(BAL_RADIX * n_tiles); w.totals = c.take<uint32_t>(SCAN_SEGMENTS);
    // touched and recv_any are next to each other: one memset clears both
    w.touched = c.take<uint8_t>(2 * n_acct); w.recv_any = w.touched ? w.touched + n_acct : nullptr;
    w.rflags = c.take<uint8_t>(n_acct); w.present = c.take<uint8_t>(n_acct); w.ok = c.take<uint8_t>(np);
    w.has = c.take<uint8_t>(2 * n_acct); w.head = c.take<uint8_t>(ne);
    w.dec = c.take<Ext>(np); w.pts = c.take<Ext>(np);
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
    return c.off;
}

static unsigned grid(const zk_ctx *, size_t n) { return (unsigned)(n ? (n + BT - 1) / BT : 1); }

// radix passes over the bits of the largest key, 2 n_accounts
static int key_passes(size_t n_acct) {
    int bits = 0;
    while (bits < 32 && ((2 * (uint64_t)n_acct) >> bits)) bits++;
    return bits <= BAL_RADIX_BITS ? 1 : (bits + BAL_RADIX_BITS - 1) / BAL_RADIX_BITS;
}

int zk_bal_prefix_sum(zk_ctx *ctx, uint32_t *c, size_t n, uint32_t *totals) {
    // up to SCAN_SEGMENTS segments of at least SCAN_MIN_SEG counters: their sums, a scan of the sums, each segment's scan
    cudaStream_t st = ctx->stream;
    size_t segs = (n + SCAN_MIN_SEG - 1) / SCAN_MIN_SEG;
    segs = segs < SCAN_SEGMENTS ? segs : SCAN_SEGMENTS;
    const size_t seg = (n + segs - 1) / segs;
    if (segs > 1) {
        k_bal_counter_sums<<<(unsigned)segs, SCAN_THREADS, 0, st>>>(c, n, seg, totals);
        k_bal_counter_scan<<<1, SCAN_THREADS, 0, st>>>(totals, segs, segs, nullptr);
    }
    k_bal_counter_scan<<<(unsigned)segs, SCAN_THREADS, 0, st>>>(c, n, seg, segs > 1 ? totals : nullptr);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

int zk_bal_sort(zk_ctx *ctx, size_t ne, size_t n_acct, uint32_t *keys0, uint32_t *keys1, uint32_t *vals0, uint32_t *vals1, uint32_t *hist,
                uint32_t *totals, const uint32_t **keys, const uint32_t **vals) {
    // stable sort of the elements by key.  (The MSM's counting sorts in msm.cuh scatter with atomicAdd cursors, so the
    // order inside a bucket is not kept; here the order inside an account is the transaction order the scan needs.)
    // One thread walks BAL_SORT_TILE consecutive elements in order, counting and then placing them through its own
    // column of the [digit][tile] counters in global memory.
    cudaStream_t st = ctx->stream;
    const size_t n_tiles = (ne + BAL_SORT_TILE - 1) / BAL_SORT_TILE;
    const int passes = key_passes(n_acct);
    uint32_t *kin = keys0, *vin = nullptr, *kout = keys1, *vout = vals1;
    for (int p = 0; p < passes; p++) {
        ZK_CUDA(cudaMemsetAsync(hist, 0, sizeof(uint32_t) * BAL_RADIX * n_tiles, st));
        k_bal_radix_hist<<<grid(ctx, n_tiles), BT, 0, st>>>(ne, kin, BAL_RADIX_BITS * p, n_tiles, hist);
        ZK_TRY(zk_bal_prefix_sum(ctx, hist, BAL_RADIX * n_tiles, totals));
        k_bal_radix_scatter<<<grid(ctx, n_tiles), BT, 0, st>>>(ne, kin, vin, BAL_RADIX_BITS * p, n_tiles, hist, kout, vout);
        kin = kout; vin = vout;
        kout = kin == keys1 ? keys0 : keys1;
        vout = vin == vals1 ? vals0 : vals1;
    }
    *keys = kin;
    *vals = vin;
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

int zk_bal_scan(zk_ctx *ctx, const uint32_t *keys, const uint32_t *vals, const Pair *delta, size_t L, const size_t *lvl_n,
                Pair *const *lvl_agg, Pair *const *lvl_out, uint8_t *const *lvl_head) {
    // segmented exclusive scan: up the levels, then down
    cudaStream_t st = ctx->stream;
    const size_t ne = lvl_n[0];
    k_bal_heads<<<grid(ctx, ne), BT, 0, st>>>(ne, keys, lvl_head[0]);
    for (size_t l = 0; l + 1 < L; l++)
        k_bal_scan_up<<<grid(ctx, lvl_n[l + 1]), BT, 0, st>>>(lvl_n[l], l ? lvl_agg[l] : delta, l ? nullptr : vals, lvl_head[l],
                                                              lvl_agg[l + 1], lvl_head[l + 1]);
    for (size_t l = L; l-- > 0;)
        k_bal_scan_down<<<grid(ctx, (lvl_n[l] + BAL_SCAN_CHUNK - 1) / BAL_SCAN_CHUNK), BT, 0, st>>>(
            lvl_n[l], l ? lvl_agg[l] : delta, l ? nullptr : vals, lvl_head[l], l + 1 < L ? lvl_out[l + 1] : nullptr, l == 0, lvl_out[l]);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

static int run_block(zk_ctx *ctx, size_t n_acct, const uint8_t *balances, const uint8_t *pendings, const uint8_t *acct_flags, size_t n_tx,
                     const uint32_t *sender, const uint32_t *recipient, const uint8_t *tx_points, const uint8_t *applied,
                     uint8_t *balance_sender, uint8_t *balance_after, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings,
                     uint8_t *new_flags, DevBuf &buf) {
    cudaStream_t st = ctx->stream;
    BalWork w;
    Carve sizing;
    ZK_TRY(buf.reserve(carve(sizing, w, n_tx, n_acct)));
    Carve c;
    c.base = buf.as<uint8_t>();
    carve(c, w, n_tx, n_acct);
    const size_t ne = 2 * n_tx, np = 4 * n_tx + 4 * n_acct;
    const uint32_t na = (uint32_t)n_acct;

    ZK_CUDA(cudaMemsetAsync(w.touched, 0, 2 * n_acct, st));
    ZK_CUDA(cudaMemsetAsync(w.has, 0, 2 * n_acct, st));
    // the failing-account word: an error word of the context, reported (and cleared) by zk_check_err_flag
    uint32_t *bad = reinterpret_cast<uint32_t *>(ctx->d_err + ZK_ERR_SLOT_ACCOUNT);
    if (n_tx) k_bal_touch<<<grid(ctx, n_tx), BT, 0, st>>>(n_tx, na, sender, recipient, w.keys0, w.touched);
    k_bal_decode<<<grid(ctx, np), BT, 0, st>>>(np, n_tx, tx_points, balances, pendings, acct_flags, w.touched, w.dec, w.ok);
    if (n_tx) k_bal_tx<<<grid(ctx, n_tx), BT, 0, st>>>(n_tx, na, sender, recipient, applied, w.dec, w.ok, w.delta, tx_status, w.recv_any);
    k_bal_account<<<grid(ctx, n_acct), BT, 0, st>>>(n_acct, n_tx, acct_flags, w.touched, w.dec, w.ok, w.roll_b, w.roll_p, w.rflags, bad);
    ZK_CUDA(cudaGetLastError());
    if (n_tx) {
        const uint32_t *keys, *vals;
        ZK_TRY(zk_bal_sort(ctx, ne, n_acct, w.keys0, w.keys1, w.vals0, w.vals1, w.hist, w.totals, &keys, &vals));
        ZK_TRY(zk_bal_scan(ctx, keys, vals, w.delta, w.lvl_n.size(), w.lvl_n.data(), w.lvl_agg.data(), w.lvl_out.data(), w.lvl_head.data()));
        k_bal_tx_points<<<grid(ctx, ne), BT, 0, st>>>(ne, na, keys, vals, w.excl, w.delta, w.roll_b, w.rflags, tx_status, w.pts, w.tot, w.has);
        ZK_CUDA(cudaGetLastError());
    }
    k_bal_acct_points<<<grid(ctx, n_acct), BT, 0, st>>>(n_acct, n_tx, w.touched, w.roll_b, w.roll_p, w.rflags, w.tot, w.has, w.recv_any,
                                                        w.pts, w.present);
    k_bal_encode<<<grid(ctx, (np + BAL_ENC_CHUNK - 1) / BAL_ENC_CHUNK), BT, 0, st>>>(np, w.pts, w.prefix, w.enc);
    if (n_tx) k_bal_finish_tx<<<grid(ctx, n_tx), BT, 0, st>>>(n_tx, tx_status, w.enc, balance_sender, balance_after);
    k_bal_finish_acct<<<grid(ctx, n_acct), BT, 0, st>>>(n_acct, n_tx, w.touched, balances, pendings, acct_flags, w.present, w.enc,
                                                        new_balances, new_pendings, new_flags);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

static int check_args(const char *fn, zk_ctx *ctx, size_t n_accounts, const void *balances, const void *pendings, const void *acct_flags,
                      size_t n_tx, const void *sender, const void *recipient, const void *tx_points, const void *applied,
                      const void *balance_sender, const void *balance_after, const void *tx_status, const void *new_balances,
                      const void *new_pendings, const void *new_flags) {
    if (!ctx || (n_accounts && (!balances || !pendings || !acct_flags || !new_balances || !new_pendings || !new_flags)) ||
        (n_tx && (!sender || !recipient || !tx_points || !applied || !balance_sender || !balance_after || !tx_status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (n_accounts > BAL_MAX || n_tx > BAL_MAX) {
        zk_set_error("%s: n_accounts = %zu, n_tx = %zu: each must be at most %u", fn, n_accounts, n_tx, BAL_MAX);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

extern "C" int zk_balances_confidential_block_device(zk_ctx *ctx, size_t n_accounts, const uint8_t *d_balances, const uint8_t *d_pendings,
                                                     const uint8_t *d_acct_flags, size_t n_tx, const uint32_t *d_sender,
                                                     const uint32_t *d_recipient, const uint8_t *d_tx_points, const uint8_t *d_applied,
                                                     uint8_t *d_balance_sender, uint8_t *d_balance_after, uint8_t *d_tx_status,
                                                     uint8_t *d_new_balances, uint8_t *d_new_pendings, uint8_t *d_new_flags) {
    ZK_TRY(check_args("zk_balances_confidential_block_device", ctx, n_accounts, d_balances, d_pendings, d_acct_flags, n_tx, d_sender,
                      d_recipient, d_tx_points, d_applied, d_balance_sender, d_balance_after, d_tx_status, d_new_balances, d_new_pendings,
                      d_new_flags));
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return run_block(ctx, n_accounts, d_balances, d_pendings, d_acct_flags, n_tx, d_sender, d_recipient, d_tx_points, d_applied,
                     d_balance_sender, d_balance_after, d_tx_status, d_new_balances, d_new_pendings, d_new_flags, ctx->bal);
}

extern "C" int zk_balances_confidential_block(zk_ctx *ctx, size_t n_accounts, const uint8_t *balances, const uint8_t *pendings,
                                              const uint8_t *acct_flags, size_t n_tx, const uint32_t *sender, const uint32_t *recipient,
                                              const uint8_t *tx_points, const uint8_t *applied, uint8_t *balance_sender,
                                              uint8_t *balance_after, uint8_t *tx_status, uint8_t *new_balances, uint8_t *new_pendings,
                                              uint8_t *new_flags) {
    ZK_TRY(check_args("zk_balances_confidential_block", ctx, n_accounts, balances, pendings, acct_flags, n_tx, sender, recipient,
                      tx_points, applied, balance_sender, balance_after, tx_status, new_balances, new_pendings, new_flags));
    if (!n_accounts && !n_tx) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *b, *p, *f, *tp, *ap;
    const uint32_t *s, *r;
    uint8_t *bs, *ba, *ts, *nb, *npd, *nf;
    Stage io;
    io.in(balances, b, 64 * n_accounts); io.in(pendings, p, 64 * n_accounts); io.in(acct_flags, f, n_accounts);
    io.in(sender, s, n_tx); io.in(recipient, r, n_tx); io.in(tx_points, tp, 128 * n_tx); io.in(applied, ap, n_tx);
    io.out(balance_sender, bs, 64 * n_tx);
    io.inout(balance_after, ba, 64 * n_tx);       // only the applied transactions' entries are written
    io.out(tx_status, ts, n_tx);
    io.out(new_balances, nb, 64 * n_accounts); io.out(new_pendings, npd, 64 * n_accounts); io.out(new_flags, nf, n_accounts);
    ZK_TRY(io.up(ctx));
    ZK_TRY(run_block(ctx, n_accounts, b, p, f, n_tx, s, r, tp, ap, bs, ba, ts, nb, npd, nf, ctx->bal));
    ZK_TRY(io.down(ctx));
    return zk_check_err_flag(ctx);     // synchronises the stream; ZK_ERR_DECODE names a touched account that failed to read
}
