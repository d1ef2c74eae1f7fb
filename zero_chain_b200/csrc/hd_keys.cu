// Wallet keys on the device (hd_keys.cuh): zk_xsk_master_batch, zk_xsk_derive_batch and zk_xpgk_derive_batch, each with
// its _device form.  The master call runs one thread per seed.  The derive calls first mark the parents some in-range row
// names, then read each marked parent once in a pass with one thread per parent (its pgk encoding and tag, and for an xpgk
// its Niels form, parked in a workspace of the context), then run one thread per row.
//
// Like tx_build.cu, the translation unit holds only Fr / Fs arithmetic and is compiled with everything inlined (ZK_HOT).
#define ZK_HOT 1
#include "internal.h"
#include "hd_keys.cuh"

using namespace zkhd;

constexpr int HT = 128;             // threads per block
constexpr int HD_BLOCKS_PER_SM = 8; // grid cap: larger batches loop over the grid
constexpr size_t HD_MAX_ROWS = (size_t)1 << 26, HD_MAX_PARENTS = (size_t)1 << 24;

#define HD_ROWS(i, n) for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (size_t)gridDim.x * blockDim.x)
static __device__ __forceinline__ uint8_t *hd_at(uint8_t *base, size_t i, int size) { return base ? base + (size_t)size * i : nullptr; }

// seed i = seeds[off[i] - base .. off[i + 1] - base); xpgks, dks and eks may be NULL
static __global__ void __launch_bounds__(HT) k_hd_master(size_t n, const uint8_t *__restrict__ seeds, const uint64_t *__restrict__ off,
                                                         uint64_t base, uint8_t *__restrict__ xsks, uint8_t *__restrict__ xpgks,
                                                         uint8_t *__restrict__ dks, uint8_t *__restrict__ eks) {
    HD_ROWS(i, n) {
        const uint64_t o0 = off[i] - base, o1 = off[i + 1] - base;
        xsk_master(seeds + o0, o1 - o0, xsks + (size_t)HD_XK_BYTES * i, hd_at(xpgks, i, HD_XK_BYTES), hd_at(dks, i, 32), hd_at(eks, i, 32));
    }
}

// one thread per row: flags the parent an in-range index names (named[] zeroed before)
static __global__ void __launch_bounds__(HT) k_hd_named(size_t n, const uint32_t *__restrict__ parent_idx, size_t n_parents,
                                                        uint8_t *__restrict__ named) {
    HD_ROWS(i, n) {
        const uint32_t p = parent_idx[i];
        if (p < n_parents) named[p] = 1;
    }
}

// one thread per parent: a named parent is read once, whatever number of rows name it; the others are left alone.
// pstatus[p]: 0, or 1 for an sk >= r_J (reported through the context's error word)
static __global__ void __launch_bounds__(HT) k_hd_xsk_parents(size_t n_parents, const uint8_t *__restrict__ parents,
                                                              const uint8_t *__restrict__ named, uint32_t *__restrict__ penc,
                                                              uint32_t *__restrict__ ptag, uint8_t *__restrict__ pstatus, int *not_canonical) {
    HD_ROWS(p, n_parents) {
        if (!named[p]) continue;
        uint32_t pgk[8], tag = 0;
        const bool ok = xsk_parent(parents + (size_t)HD_XK_BYTES * p, pgk, tag);
        pstatus[p] = !ok;
        if (!ok) {
            atomicExch(not_canonical, 1);
            continue;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) penc[8 * p + k] = pgk[k];
        ptag[p] = tag;
    }
}

static __global__ void __launch_bounds__(HT) k_hd_xsk_rows(size_t n, const uint8_t *__restrict__ parents, size_t n_parents,
                                                           const uint32_t *__restrict__ parent_idx, const uint32_t *__restrict__ child_idx,
                                                           const uint32_t *__restrict__ penc, const uint32_t *__restrict__ ptag,
                                                           const uint8_t *__restrict__ pstatus, uint8_t *__restrict__ xsks,
                                                           uint8_t *__restrict__ xpgks, uint8_t *__restrict__ dks, uint8_t *__restrict__ eks,
                                                           uint8_t *__restrict__ status) {
    HD_ROWS(i, n) {
        const int st = xsk_row(parents, n_parents, parent_idx[i], child_idx[i], penc, ptag, pstatus, xsks + (size_t)HD_XK_BYTES * i,
                               hd_at(xpgks, i, HD_XK_BYTES), hd_at(dks, i, 32), hd_at(eks, i, 32));
        if (st >= 0) status[i] = (uint8_t)st;
    }
}

// one thread per parent: ProofGenerationKey::read of each named parent once; pstatus[p] its zk_jubjub_into_xy code
static __global__ void __launch_bounds__(HT) k_hd_xpgk_parents(size_t n_parents, const uint8_t *__restrict__ parents,
                                                               const uint8_t *__restrict__ named, uint32_t *__restrict__ penc,
                                                               uint32_t *__restrict__ ptag, uint32_t *__restrict__ pniels,
                                                               uint8_t *__restrict__ pstatus) {
    HD_ROWS(p, n_parents) {
        if (!named[p]) continue;
        uint32_t pgk[8], niels[TB_ENTRY_WORDS], tag = 0;
        const int st = xpgk_parent(parents + (size_t)HD_XK_BYTES * p, pgk, niels, tag);
        pstatus[p] = (uint8_t)st;
        if (st != JJ_OK) continue;
#pragma unroll
        for (int k = 0; k < 8; k++) penc[8 * p + k] = pgk[k];
#pragma unroll
        for (int k = 0; k < TB_ENTRY_WORDS; k++) pniels[TB_ENTRY_WORDS * p + k] = niels[k];
        ptag[p] = tag;
    }
}

static __global__ void __launch_bounds__(HT) k_hd_xpgk_rows(size_t n, const uint8_t *__restrict__ parents, size_t n_parents,
                                                            const uint32_t *__restrict__ parent_idx, const uint32_t *__restrict__ child_idx,
                                                            const uint32_t *__restrict__ penc, const uint32_t *__restrict__ ptag,
                                                            const uint32_t *__restrict__ pniels, const uint8_t *__restrict__ pstatus,
                                                            uint8_t *__restrict__ xpgks, uint8_t *__restrict__ dks, uint8_t *__restrict__ eks,
                                                            uint8_t *__restrict__ status) {
    HD_ROWS(i, n)
        status[i] = (uint8_t)xpgk_row(parents, n_parents, parent_idx[i], child_idx[i], penc, ptag, pniels, pstatus, xpgks + (size_t)HD_XK_BYTES * i,
                                      hd_at(dks, i, 32), hd_at(eks, i, 32));
}

static unsigned grid(const zk_ctx *ctx, size_t n) {
    const size_t cap = (size_t)(ctx->sm_count > 0 ? ctx->sm_count : 1) * HD_BLOCKS_PER_SM;
    return (unsigned)((n + HT - 1) / HT < cap ? (n + HT - 1) / HT : cap);
}

// ---- host-side checks -------------------------------------------------------------------------------------------------
static int check_offsets(const char *fn, size_t n, const uint64_t *off) {
    for (size_t i = 0; i < n; i++)
        if (off[i + 1] < off[i]) {
            zk_set_error("%s: off[%zu] = %llu > off[%zu] = %llu", fn, i, (unsigned long long)off[i], i + 1, (unsigned long long)off[i + 1]);
            return ZK_ERR_INVALID;
        }
    return ZK_OK;
}
static int check_sizes(const char *fn, size_t n_parents, size_t n) {
    if (n > HD_MAX_ROWS || n_parents > HD_MAX_PARENTS) {
        zk_set_error("%s: n = %zu, n_parents = %zu; at most 2^26 rows and 2^24 parents", fn, n, n_parents);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}
// SpendingKey::read of every parent an in-range row names: ZK_ERR_NOT_CANONICAL naming the lowest such parent whose sk >= r_J
static int check_parents(const char *fn, size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *parent_idx) {
    static const uint32_t r_j[8] = {0xd6f72cb7u, 0xd0970e5eu, 0xccc81082u, 0xa6682093u, 0x01343b00u, 0x06673b01u, 0x6533afa9u, 0x0e7db4eau};
    size_t bad = n_parents;
    for (size_t i = 0; i < n; i++) {
        const size_t p = parent_idx[i];
        if (p >= bad) continue;
        const uint8_t *b = parents + (size_t)HD_XK_BYTES * p + HD_KEY;
        bool lt = false;
        for (int k = 31; k >= 0; k--) {
            const uint8_t m = (uint8_t)(r_j[k / 4] >> (8 * (k % 4)));
            if (b[k] != m) { lt = b[k] < m; break; }
        }
        if (!lt) bad = p;
    }
    if (bad == n_parents) return ZK_OK;
    zk_set_error("%s: parents[%zu] has sk >= r_J (SpendingKey::read fails)", fn, bad);
    return ZK_ERR_NOT_CANONICAL;
}

// ---- zk_xsk_master_batch --------------------------------------------------------------------------------------------------
extern "C" int zk_xsk_master_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_seeds, const uint64_t *d_seed_off, uint8_t *d_xsks,
                                          uint8_t *d_xpgks, uint8_t *d_dks, uint8_t *d_eks) {
    if (!ctx || (n && (!d_seeds || !d_seed_off || !d_xsks))) {
        zk_set_error("zk_xsk_master_batch_device: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    k_hd_master<<<grid(ctx, n), HT, 0, ctx->stream>>>(n, d_seeds, d_seed_off, 0, d_xsks, d_xpgks, d_dks, d_eks);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_xsk_master_batch(zk_ctx *ctx, size_t n, const uint8_t *seeds, const uint64_t *seed_off, uint8_t *xsks, uint8_t *xpgks,
                                   uint8_t *dks, uint8_t *eks) {
    static const char *fn = "zk_xsk_master_batch";
    if (!ctx || (n && (!seeds || !seed_off || !xsks))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(check_offsets(fn, n, seed_off));
    ZK_TRY(zk_use_device(ctx));
    const uint64_t base = seed_off[0];
    const uint8_t *d_seeds;
    const uint64_t *d_off;
    uint8_t *d_xsks, *d_xpgks, *d_dks, *d_eks;
    Stage io;
    io.in(seed_off, d_off, n + 1); io.in(seeds + base, d_seeds, seed_off[n] - base);
    io.out(xsks, d_xsks, HD_XK_BYTES * n); io.out(xpgks, d_xpgks, HD_XK_BYTES * n); io.out(dks, d_dks, 32 * n); io.out(eks, d_eks, 32 * n);
    ZK_TRY(io.up(ctx));
    k_hd_master<<<grid(ctx, n), HT, 0, ctx->stream>>>(n, d_seeds, d_off, base, d_xsks, d_xpgks, d_dks, d_eks);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

// ---- the derive calls: the named pass, the parent pass, the row pass ------------------------------------------------------
struct HdParents {
    uint8_t *named, *status;
    uint32_t *enc, *tag, *niels;
};
static int hd_workspace(zk_ctx *ctx, size_t n_parents, bool with_niels, size_t n, const uint32_t *parent_idx, HdParents &w) {
    Carve sizing;
    sizing.take<uint8_t>(n_parents); sizing.take<uint8_t>(n_parents); sizing.take<uint32_t>(8 * n_parents); sizing.take<uint32_t>(n_parents);
    sizing.take<uint32_t>(with_niels ? TB_ENTRY_WORDS * n_parents : 0);
    ZK_TRY(ctx->hd.reserve(sizing.off));
    Carve c{ctx->hd.as<uint8_t>(), 0};
    w.named = c.take<uint8_t>(n_parents); w.status = c.take<uint8_t>(n_parents);
    w.enc = c.take<uint32_t>(8 * n_parents); w.tag = c.take<uint32_t>(n_parents);
    w.niels = c.take<uint32_t>(with_niels ? TB_ENTRY_WORDS * n_parents : 0);
    if (n_parents) {
        ZK_CUDA(cudaMemsetAsync(w.named, 0, n_parents, ctx->stream));
        k_hd_named<<<grid(ctx, n), HT, 0, ctx->stream>>>(n, parent_idx, n_parents, w.named);
        ZK_CUDA(cudaGetLastError());
    }
    return ZK_OK;
}

static int launch_xsk(zk_ctx *ctx, size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *parent_idx, const uint32_t *child_idx,
                      uint8_t *xsks, uint8_t *xpgks, uint8_t *dks, uint8_t *eks, uint8_t *status) {
    HdParents w;
    ZK_TRY(hd_workspace(ctx, n_parents, false, n, parent_idx, w));
    if (n_parents) {
        k_hd_xsk_parents<<<grid(ctx, n_parents), HT, 0, ctx->stream>>>(n_parents, parents, w.named, w.enc, w.tag, w.status, ctx->d_err);
        ZK_CUDA(cudaGetLastError());
    }
    k_hd_xsk_rows<<<grid(ctx, n), HT, 0, ctx->stream>>>(n, parents, n_parents, parent_idx, child_idx, w.enc, w.tag, w.status, xsks, xpgks, dks,
                                                        eks, status);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

static int launch_xpgk(zk_ctx *ctx, size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *parent_idx, const uint32_t *child_idx,
                       uint8_t *xpgks, uint8_t *dks, uint8_t *eks, uint8_t *status) {
    HdParents w;
    ZK_TRY(hd_workspace(ctx, n_parents, true, n, parent_idx, w));
    if (n_parents) {
        k_hd_xpgk_parents<<<grid(ctx, n_parents), HT, 0, ctx->stream>>>(n_parents, parents, w.named, w.enc, w.tag, w.niels, w.status);
        ZK_CUDA(cudaGetLastError());
    }
    k_hd_xpgk_rows<<<grid(ctx, n), HT, 0, ctx->stream>>>(n, parents, n_parents, parent_idx, child_idx, w.enc, w.tag, w.niels, w.status, xpgks,
                                                         dks, eks, status);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

// ---- zk_xsk_derive_batch --------------------------------------------------------------------------------------------------
extern "C" int zk_xsk_derive_batch_device(zk_ctx *ctx, size_t n_parents, const uint8_t *d_parents, size_t n, const uint32_t *d_parent_idx,
                                          const uint32_t *d_child_idx, uint8_t *d_xsks, uint8_t *d_xpgks, uint8_t *d_dks, uint8_t *d_eks,
                                          uint8_t *d_status) {
    static const char *fn = "zk_xsk_derive_batch_device";
    if (!ctx || (n_parents && !d_parents) || (n && (!d_parent_idx || !d_child_idx || !d_xsks || !d_status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    ZK_TRY(check_sizes(fn, n_parents, n));
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return launch_xsk(ctx, n_parents, d_parents, n, d_parent_idx, d_child_idx, d_xsks, d_xpgks, d_dks, d_eks, d_status);
}

extern "C" int zk_xsk_derive_batch(zk_ctx *ctx, size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *parent_idx,
                                   const uint32_t *child_idx, uint8_t *xsks, uint8_t *xpgks, uint8_t *dks, uint8_t *eks, uint8_t *status) {
    static const char *fn = "zk_xsk_derive_batch";
    if (!ctx || (n_parents && !parents) || (n && (!parent_idx || !child_idx || !xsks || !status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    ZK_TRY(check_sizes(fn, n_parents, n));
    if (!n) return ZK_OK;
    ZK_TRY(check_parents(fn, n_parents, parents, n, parent_idx));
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d_parents;
    const uint32_t *d_pidx, *d_cidx;
    uint8_t *d_xsks, *d_xpgks, *d_dks, *d_eks, *d_st;
    Stage io;
    io.in(parents, d_parents, HD_XK_BYTES * n_parents); io.in(parent_idx, d_pidx, n); io.in(child_idx, d_cidx, n);
    io.out(xsks, d_xsks, HD_XK_BYTES * n); io.out(xpgks, d_xpgks, HD_XK_BYTES * n); io.out(dks, d_dks, 32 * n); io.out(eks, d_eks, 32 * n);
    io.out(status, d_st, n);
    ZK_TRY(io.up(ctx));
    ZK_TRY(launch_xsk(ctx, n_parents, d_parents, n, d_pidx, d_cidx, d_xsks, d_xpgks, d_dks, d_eks, d_st));
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

// ---- zk_xpgk_derive_batch -------------------------------------------------------------------------------------------------
extern "C" int zk_xpgk_derive_batch_device(zk_ctx *ctx, size_t n_parents, const uint8_t *d_parents, size_t n, const uint32_t *d_parent_idx,
                                           const uint32_t *d_child_idx, uint8_t *d_xpgks, uint8_t *d_dks, uint8_t *d_eks, uint8_t *d_status) {
    static const char *fn = "zk_xpgk_derive_batch_device";
    if (!ctx || (n_parents && !d_parents) || (n && (!d_parent_idx || !d_child_idx || !d_xpgks || !d_status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    ZK_TRY(check_sizes(fn, n_parents, n));
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return launch_xpgk(ctx, n_parents, d_parents, n, d_parent_idx, d_child_idx, d_xpgks, d_dks, d_eks, d_status);
}

extern "C" int zk_xpgk_derive_batch(zk_ctx *ctx, size_t n_parents, const uint8_t *parents, size_t n, const uint32_t *parent_idx,
                                    const uint32_t *child_idx, uint8_t *xpgks, uint8_t *dks, uint8_t *eks, uint8_t *status) {
    static const char *fn = "zk_xpgk_derive_batch";
    if (!ctx || (n_parents && !parents) || (n && (!parent_idx || !child_idx || !xpgks || !status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    ZK_TRY(check_sizes(fn, n_parents, n));
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d_parents;
    const uint32_t *d_pidx, *d_cidx;
    uint8_t *d_xpgks, *d_dks, *d_eks, *d_st;
    Stage io;
    io.in(parents, d_parents, HD_XK_BYTES * n_parents); io.in(parent_idx, d_pidx, n); io.in(child_idx, d_cidx, n);
    io.out(xpgks, d_xpgks, HD_XK_BYTES * n); io.out(dks, d_dks, 32 * n); io.out(eks, d_eks, 32 * n); io.out(status, d_st, n);
    ZK_TRY(io.up(ctx));
    ZK_TRY(launch_xpgk(ctx, n_parents, d_parents, n, d_pidx, d_cidx, d_xpgks, d_dks, d_eks, d_st));
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}
