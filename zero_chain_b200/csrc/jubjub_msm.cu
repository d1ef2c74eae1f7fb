// Jubjub multi-scalar multiplication on the device (jubjub_msm.cuh) and RedJubjub batch verification built on it:
// zk_jubjub_msm, zk_redjubjub_batch_verify and its _device form.
//
// One call runs on the context's stream:
//   bases        k_jm_read_points (thread per encoding: Point::read, Niels form) or k_rj_batch_prep (thread per entry:
//                BLAKE2b, two Point::reads, the scalars z and z c, a block sum of z S) + k_rj_batch_last (the -P_G term)
//   digits/sort  k_msm_digits, k_tile_hist, k_col_scan, k_scatter of msm.cuh with one sort domain per window
//   buckets      k_jm_task_counts + scan, k_jm_accumulate (thread per run of <= JM_RUN entries), k_jm_combine /
//                k_jm_combine_warp (a bucket's runs; warp per bucket with more than JM_COMB_SERIAL runs)
//   reduction    k_jm_slices (thread per slice of L buckets), k_jm_windows (thread per window), k_jm_horner (one thread)
//   result       k_jm_encode (Point::write) or k_rj_batch_verdict (three doublings, the identity test, the first rejection)
// The buffers live in one grow-only arena of the context (ctx->jm).
//
// Like jubjub.cu, the translation unit holds only Fr / Fs arithmetic and is compiled with everything inlined (ZK_HOT).
#define ZK_HOT 1
#include "internal.h"
#include "msm.cuh"
#include "jubjub_msm.cuh"

using namespace zkjm;

constexpr int JT = 128;                      // threads per block of the per-item kernels
constexpr int JM_BLOCKS_PER_SM = 8;          // grid cap of the per-entry kernel: larger batches loop over the grid
constexpr uint32_t JM_COMB_SERIAL = 32;      // runs per bucket folded by one thread; more go to a warp
constexpr size_t JM_MAX_POINTS = (size_t)1 << 26;   // W n entries must stay below 2^32
constexpr uint8_t RJ_BAD_Z = 5;              // _device form only: a z_i >= r_J
constexpr unsigned long long JM_NO_BAD = ~0ull;

static __device__ __forceinline__ void load_le_bytes(const uint8_t *b, uint32_t *w, int n) {
#pragma unroll
    for (int i = 0; i < n; i++)     // byte loads: a device pointer passed in by the caller need not be word aligned
        w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
}
static __device__ __forceinline__ Fs fs_shfl_down(const Fs &a, int o) {
    Fs r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.l[i] = __shfl_down_sync(0xffffffffu, a.l[i], o);
    return r;
}
// the sum mod r_J of every thread's canonical v, in thread 0 (blockDim.x a multiple of 32, at most 1024)
static __device__ __forceinline__ Fs fs_block_sum(Fs v) {
    __shared__ uint32_t wsum[32][8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = v + fs_shfl_down(v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int i = 0; i < 8; i++) wsum[warp][i] = v.l[i];
    __syncthreads();
    if (threadIdx.x == 0)
        for (int k = 1; k < (int)(blockDim.x >> 5); k++) {
            Fs u;
#pragma unroll
            for (int i = 0; i < 8; i++) u.l[i] = wsum[k][i];
            v = v + u;
        }
    return v;
}

// ---- bases ---------------------------------------------------------------------------------------------------------------
static __global__ void __launch_bounds__(JT) k_jm_read_points(size_t n, const uint8_t *__restrict__ enc, uint32_t *__restrict__ niels,
                                                              unsigned long long *__restrict__ bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t e[8];
    load_le_bytes(enc + 32 * i, e, 8);
    Niels q;
    if (jm_read_niels(e, q) != JJ_OK) atomicMin(bad, (unsigned long long)i);
    jm_niels_store(niels + (size_t)JM_NIELS_WORDS * i, q);
}

// entry i: bases R_i at i and vk_i at n + i, scalars z_i and z_i c_i likewise; part[block] = the block's sum of z_i S_i.
// A rejected entry records (i << 3 | code) in *bad with atomicMin, so the lowest rejected index wins.
static __global__ void __launch_bounds__(JT) k_rj_batch_prep(size_t n, const uint8_t *__restrict__ vks, const uint8_t *__restrict__ sigs,
                                                             const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base,
                                                             const uint8_t *__restrict__ zs, uint32_t *__restrict__ niels,
                                                             uint32_t *__restrict__ scalars, uint32_t *__restrict__ part,
                                                             unsigned long long *__restrict__ bad) {
    Fs sum = Fs::zero();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t vk[8], sig[16], z[8];
        load_le_bytes(zs + 32 * i, z, 8);
        load_le_bytes(vks + 32 * i, vk, 8);
        load_le_bytes(sigs + 64 * i, sig, 16);
        const uint64_t o0 = off[i] - base, o1 = off[i + 1] - base;
        Niels nr, nvk;
        Fs zc, zsi;
        int code;
        {
            Fs zf;
#pragma unroll
            for (int k = 0; k < 8; k++) zf.l[k] = z[k];
            code = Fs::canonical_lt_mod(zf) ? rj_batch_entry(vk, sig, msgs + o0, o1 - o0, z, nr, nvk, zc, zsi) : RJ_BAD_Z;
        }
        if (code != zkrj::RJ_OK) {
            atomicMin(bad, ((unsigned long long)i << 3) | (unsigned long long)code);
            nr = zkrj::niels_identity(); nvk = nr; zc = Fs::zero(); zsi = zc;
        }
        jm_niels_store(niels + (size_t)JM_NIELS_WORDS * i, nr);
        jm_niels_store(niels + (size_t)JM_NIELS_WORDS * (n + i), nvk);
        Fs zr;
#pragma unroll
        for (int k = 0; k < 8; k++) zr.l[k] = code == zkrj::RJ_OK ? z[k] : 0u;
        jm_store_words(scalars + 8 * i, zr.l, 2);
        jm_store_words(scalars + 8 * (n + i), zc.l, 2);
        sum = sum + zsi;
    }
    sum = fs_block_sum(sum);
    if (threadIdx.x == 0) jm_store_words(part + 8 * (size_t)blockIdx.x, sum.l, 2);
}
// the last term: base -P_G at 2n with scalar sum_i z_i S_i (the block partials summed)
static __global__ void __launch_bounds__(256) k_rj_batch_last(size_t n, uint32_t n_part, const uint32_t *__restrict__ part,
                                                              uint32_t *__restrict__ niels, uint32_t *__restrict__ scalars) {
    Fs v = Fs::zero();
    for (uint32_t k = threadIdx.x; k < n_part; k += blockDim.x) {
        Fs u;
        jm_load_words(part + 8 * (size_t)k, u.l, 2);
        v = v + u;
    }
    v = fs_block_sum(v);
    if (threadIdx.x == 0) {
        jm_niels_store(niels + (size_t)JM_NIELS_WORDS * 2 * n, zkrj::niels_neg_pg());
        jm_store_words(scalars + 8 * 2 * n, v.l, 2);
    }
}

// ---- buckets --------------------------------------------------------------------------------------------------------------
static __global__ void k_jm_task_counts(const uint32_t *__restrict__ sizes, uint32_t NB, uint32_t *__restrict__ counts) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < NB) counts[b] = (sizes[b] + JM_RUN - 1) / JM_RUN;
}
// thread per run: the bucket's entries are split evenly over its runs
static __global__ void __launch_bounds__(JT) k_jm_accumulate(const uint32_t *__restrict__ niels, const uint32_t *__restrict__ sorted,
                                                             const uint32_t *__restrict__ bucket_off, const uint32_t *__restrict__ task_off,
                                                             uint32_t NB, uint32_t *__restrict__ partials) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= task_off[NB]) return;
    uint32_t lo = 0, hi = NB;                 // the bucket of run t: last b with task_off[b] <= t
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (task_off[mid] <= t) lo = mid; else hi = mid; }
    const uint32_t b = lo, s = t - task_off[b], nt = task_off[b + 1] - task_off[b], b0 = bucket_off[b], size = bucket_off[b + 1] - b0;
    const uint32_t len = (size + nt - 1) / nt, e0 = b0 + s * len, e1 = e0 + len < b0 + size ? e0 + len : b0 + size;
    jm_ext_store(partials + (size_t)JM_EXT_WORDS * t, jm_accumulate(niels, sorted, e0, e1 > e0 ? e1 : e0));
}
// thread per bucket: the sum of its runs; buckets with more than JM_COMB_SERIAL runs are left to k_jm_combine_warp
static __global__ void __launch_bounds__(JT) k_jm_combine(const uint32_t *__restrict__ partials, const uint32_t *__restrict__ task_off, uint32_t NB,
                                                          uint32_t *__restrict__ buckets, uint32_t *__restrict__ heavy, uint32_t *__restrict__ n_heavy) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= NB) return;
    const uint32_t t0 = task_off[b], t1 = task_off[b + 1];
    if (t1 - t0 > JM_COMB_SERIAL) { heavy[atomicAdd(n_heavy, 1u)] = b; return; }
    const Fr d2 = jj_d2();
    Ext acc = ext_identity();
#pragma unroll 1
    for (uint32_t t = t0; t < t1; t++) acc = ext_add(acc, jm_ext_load(partials + (size_t)JM_EXT_WORDS * t), d2);
    jm_ext_store(buckets + (size_t)JM_EXT_WORDS * b, acc);
}
static __device__ __forceinline__ Ext ext_shfl_down(const Ext &p, int o) {
    Ext r;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        r.x.l[i] = __shfl_down_sync(0xffffffffu, p.x.l[i], o); r.y.l[i] = __shfl_down_sync(0xffffffffu, p.y.l[i], o);
        r.z.l[i] = __shfl_down_sync(0xffffffffu, p.z.l[i], o); r.t.l[i] = __shfl_down_sync(0xffffffffu, p.t.l[i], o);
    }
    return r;
}
// fixed grid: warp w folds heavy[w], heavy[w + n_warps], ...: lanes stride over the runs, then a shuffle tree
static __global__ void __launch_bounds__(JT) k_jm_combine_warp(const uint32_t *__restrict__ partials, const uint32_t *__restrict__ task_off,
                                                               const uint32_t *__restrict__ heavy, const uint32_t *__restrict__ n_heavy,
                                                               uint32_t *__restrict__ buckets) {
    const uint32_t lane = threadIdx.x & 31, n_warps = (gridDim.x * blockDim.x) >> 5, nh = *n_heavy;
    const Fr d2 = jj_d2();
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < nh; i += n_warps) {
        const uint32_t b = heavy[i], t0 = task_off[b], t1 = task_off[b + 1];
        Ext acc = ext_identity();
#pragma unroll 1
        for (uint32_t t = t0 + lane; t < t1; t += 32) acc = ext_add(acc, jm_ext_load(partials + (size_t)JM_EXT_WORDS * t), d2);
#pragma unroll 1
        for (int o = 16; o > 0; o >>= 1) acc = ext_add(acc, ext_shfl_down(acc, o), d2);
        if (lane == 0) jm_ext_store(buckets + (size_t)JM_EXT_WORDS * b, acc);
    }
}

// ---- reduction -------------------------------------------------------------------------------------------------------------
// thread per (window, slice): S, T of slice j of window w at [w][j]
static __global__ void __launch_bounds__(JT) k_jm_slices(const uint32_t *__restrict__ buckets, uint32_t nb, uint32_t n_items, uint32_t log_L,
                                                         uint32_t *__restrict__ S, uint32_t *__restrict__ T) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_items) return;
    const uint32_t n_slices = nb >> log_L, w = g / n_slices, j = g - w * n_slices;
    Ext s, t;
    jm_slice_sums(buckets + (size_t)JM_EXT_WORDS * ((size_t)w * nb + ((size_t)j << log_L)), 1u << log_L, s, t);
    jm_ext_store(S + (size_t)JM_EXT_WORDS * g, s);
    jm_ext_store(T + (size_t)JM_EXT_WORDS * g, t);
}
static __global__ void __launch_bounds__(32) k_jm_windows(const uint32_t *__restrict__ S, const uint32_t *__restrict__ T, int W, uint32_t n_slices,
                                                          int log_L, uint32_t *__restrict__ R) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    const size_t o = (size_t)JM_EXT_WORDS * w * n_slices;
    jm_ext_store(R + (size_t)JM_EXT_WORDS * w, jm_window_sum(S + o, T + o, n_slices, log_L));
}
static __global__ void __launch_bounds__(32) k_jm_horner(const uint32_t *__restrict__ R, int W, int c, uint32_t *__restrict__ out) {
    if (threadIdx.x == 0) jm_ext_store(out, jm_horner(R, W, c));
}

// ---- results ---------------------------------------------------------------------------------------------------------------
static __global__ void __launch_bounds__(32) k_jm_encode(const uint32_t *__restrict__ result, uint32_t *__restrict__ enc) {
    if (threadIdx.x != 0) return;
    uint32_t e[8];
    jm_encode(jm_ext_load(result), e);
#pragma unroll
    for (int i = 0; i < 8; i++) enc[i] = e[i];
}
// [8] result == O, unless an entry was rejected: then its code and index
static __global__ void __launch_bounds__(32) k_rj_batch_verdict(const uint32_t *__restrict__ result, const unsigned long long *__restrict__ bad,
                                                                uint64_t n, uint8_t *__restrict__ verdict, uint64_t *__restrict__ first_bad) {
    if (threadIdx.x != 0) return;
    const unsigned long long k = *bad;
    if (k != JM_NO_BAD) {
        *verdict = (uint8_t)(k & 7u);
        if (first_bad) *first_bad = k >> 3;
        return;
    }
    const Ext acc = ext_dbl(ext_dbl(ext_dbl(jm_ext_load(result))));
    *verdict = ext_is_identity(acc) ? zkrj::RJ_OK : zkrj::RJ_BAD_EQUATION;
    if (first_bad) *first_bad = n;
}

// ---- host side ---------------------------------------------------------------------------------------------------------------
static size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }

// the shape of one MSM over n points and where its buffers sit in the arena
struct JmPlan {
    uint32_t n, nb, NB, tiles, n_slices, task_cap;
    int c, W, log_L;
    size_t o_small, o_niels, o_scalars, o_digits, o_sorted, o_hist, o_toff, o_sizes, o_boff, o_tcount, o_task, o_scan, o_part, o_buck,
        o_S, o_T, o_R, o_extra, bytes;
};
// small words at o_small: [0] digit error flag, [1] heavy-bucket count, [2..3] the first bad index (u64), [8..16) the encoding
static JmPlan jm_plan(size_t n, size_t extra) {
    JmPlan p;
    p.n = (uint32_t)n;
    int lg = 0;
    while (((size_t)2 << lg) <= n) lg++;           // floor(log2 n)
    p.c = lg - 4 < 8 ? 8 : lg - 4 > 14 ? 14 : lg - 4;
    p.W = (253 + p.c - 1) / p.c;                   // W c >= 253: the top window of a scalar < 2^252 never carries out
    p.nb = 1u << (p.c - 1);
    p.NB = (uint32_t)p.W * p.nb;
    p.tiles = (uint32_t)((n + zkmsm::TILE - 1) / zkmsm::TILE);
    p.log_L = p.c / 2;                             // L = 2^ceil((c - 1) / 2) buckets per slice
    p.n_slices = p.nb >> p.log_L;
    const size_t entries = (size_t)p.W * n;
    p.task_cap = (uint32_t)(entries / JM_RUN + (entries < p.NB ? entries : p.NB) + 1);
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t r = o; o += up256(bytes); return r; };
    p.o_small = take(64);
    p.o_niels = take((size_t)JM_NIELS_WORDS * 4 * n);
    p.o_scalars = take(32 * n);
    p.o_digits = take(4 * entries);
    p.o_sorted = take(4 * entries);
    p.o_hist = take((size_t)4 * p.W * p.tiles * p.nb);
    p.o_toff = take((size_t)4 * p.W * p.tiles * p.nb);
    p.o_sizes = take(4 * (size_t)p.NB);
    p.o_boff = take(4 * ((size_t)p.NB + 1));
    p.o_tcount = take(4 * (size_t)p.NB);
    p.o_task = take(4 * ((size_t)p.NB + 1));
    p.o_scan = take(4 * 2 * ((size_t)p.NB / zkmsm::SCAN_B + 8));
    p.o_part = take((size_t)JM_EXT_WORDS * 4 * p.task_cap);
    p.o_buck = take((size_t)JM_EXT_WORDS * 4 * p.NB);
    p.o_S = take((size_t)JM_EXT_WORDS * 4 * p.W * p.n_slices);
    p.o_T = take((size_t)JM_EXT_WORDS * 4 * p.W * p.n_slices);
    p.o_R = take((size_t)JM_EXT_WORDS * 4 * (p.W + 1));   // the windows, then the result
    p.o_extra = take(extra);
    p.bytes = o;
    return p;
}
template <class T> static T *at(zk_ctx *ctx, size_t off) { return reinterpret_cast<T *>(ctx->jm.as<uint8_t>() + off); }
static unsigned grid(size_t n, int t) { return (unsigned)((n + t - 1) / t); }

// zeroes the flags and sets the first bad index to "none"; then the bases and scalars are written by the caller
static int jm_begin(zk_ctx *ctx, const JmPlan &p) {
    ZK_TRY(ctx->jm.reserve(p.bytes));
    ZK_CUDA(cudaMemsetAsync(at<uint8_t>(ctx, p.o_small), 0, 8, ctx->stream));
    ZK_CUDA(cudaMemsetAsync(at<uint8_t>(ctx, p.o_small) + 8, 0xff, 8, ctx->stream));
    return ZK_OK;
}

// sum_i scalars[i] P_i over the bases and scalars already in the arena; the result (extended) at o_R + W points
static int jm_msm_run(zk_ctx *ctx, const JmPlan &p) {
    cudaStream_t st = ctx->stream;
    uint32_t *small = at<uint32_t>(ctx, p.o_small), *niels = at<uint32_t>(ctx, p.o_niels), *digits = at<uint32_t>(ctx, p.o_digits),
             *sorted = at<uint32_t>(ctx, p.o_sorted), *hist = at<uint32_t>(ctx, p.o_hist), *toff = at<uint32_t>(ctx, p.o_toff),
             *sizes = at<uint32_t>(ctx, p.o_sizes), *boff = at<uint32_t>(ctx, p.o_boff), *tcount = at<uint32_t>(ctx, p.o_tcount),
             *task = at<uint32_t>(ctx, p.o_task), *scan = at<uint32_t>(ctx, p.o_scan), *part = at<uint32_t>(ctx, p.o_part),
             *buck = at<uint32_t>(ctx, p.o_buck), *S = at<uint32_t>(ctx, p.o_S), *T = at<uint32_t>(ctx, p.o_T), *R = at<uint32_t>(ctx, p.o_R);
    // signed digits [window][point]; the scalars are canonical Fs, below r, so the digit kernel's check never fires
    zkmsm::k_msm_digits<<<dim3(grid(p.n, 256), 1), 256, 0, st>>>(at<uint32_t>(ctx, p.o_scalars), p.n, p.c, p.W, digits,
                                                                 reinterpret_cast<int *>(small));
    // counting sort, one domain per window: entries grouped by (window, bucket)
    const size_t shm = 4 * (size_t)p.nb;
    zkmsm::k_tile_hist<<<dim3(p.tiles, p.W), zkmsm::SORT_THREADS, shm, st>>>(digits, p.n, (int)p.nb, 0, hist, (int)p.tiles, zkmsm::TILE, false);
    zkmsm::k_col_scan<<<grid(p.NB, 256), 256, 0, st>>>(hist, toff, sizes, (int)p.nb, (int)p.tiles, p.W);
    zkmsm::exclusive_scan<false>(sizes, boff, p.NB, scan, st);
    zkmsm::k_scatter<<<dim3(p.tiles, p.W), zkmsm::SORT_THREADS, shm, st>>>(digits, p.n, (int)p.nb, toff, boff, sorted, (int)p.tiles, zkmsm::TILE);
    // buckets: runs of <= JM_RUN entries, then each bucket's runs folded
    k_jm_task_counts<<<grid(p.NB, 256), 256, 0, st>>>(sizes, p.NB, tcount);
    zkmsm::exclusive_scan<false>(tcount, task, p.NB, scan, st);
    k_jm_accumulate<<<grid(p.task_cap, JT), JT, 0, st>>>(niels, sorted, boff, task, p.NB, part);
    k_jm_combine<<<grid(p.NB, JT), JT, 0, st>>>(part, task, p.NB, buck, tcount, small + 1);   // tcount is free again: the heavy list
    k_jm_combine_warp<<<(unsigned)(ctx->sm_count > 0 ? ctx->sm_count : 1) * 4, JT, 0, st>>>(part, task, tcount, small + 1, buck);
    // sum_d d B[d] per window, then Horner over the windows
    const uint32_t n_items = (uint32_t)p.W * p.n_slices;
    k_jm_slices<<<grid(n_items, 32), 32, 0, st>>>(buck, p.nb, n_items, (uint32_t)p.log_L, S, T);
    k_jm_windows<<<grid(p.W, 32), 32, 0, st>>>(S, T, p.W, p.n_slices, p.log_L, R);
    k_jm_horner<<<1, 32, 0, st>>>(R, p.W, p.c, R + (size_t)JM_EXT_WORDS * p.W);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

// little-endian 32 bytes < r_J
static bool fs_bytes_canonical(const uint8_t *b) {
    static const uint32_t RJ[8] = {0xd6f72cb7u, 0xd0970e5eu, 0xccc81082u, 0xa6682093u, 0x01343b00u, 0x06673b01u, 0x6533afa9u, 0x0e7db4eau};
    for (int i = 7; i >= 0; i--) {
        const uint32_t w = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
        if (w != RJ[i]) return w < RJ[i];
    }
    return false;
}

extern "C" int zk_jubjub_msm(zk_ctx *ctx, size_t n, const uint8_t *points, const uint8_t *scalars, uint8_t out[32]) {
    if (!ctx || !out || (n && (!points || !scalars))) {
        zk_set_error("zk_jubjub_msm: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (n > JM_MAX_POINTS) {
        zk_set_error("zk_jubjub_msm: n = %zu > %zu", n, JM_MAX_POINTS);
        return ZK_ERR_INVALID;
    }
    for (size_t i = 0; i < n; i++)
        if (!fs_bytes_canonical(scalars + 32 * i)) {
            zk_set_error("zk_jubjub_msm: scalar %zu >= r_J", i);
            return ZK_ERR_NOT_CANONICAL;
        }
    if (!n) {                                        // the identity: y = 1, x = 0
        memset(out, 0, 32);
        out[0] = 1;
        return ZK_OK;
    }
    ZK_TRY(zk_use_device(ctx));
    const JmPlan p = jm_plan(n, 32 * n);
    ZK_TRY(jm_begin(ctx, p));
    uint8_t *d_enc = at<uint8_t>(ctx, p.o_extra);
    uint32_t *small = at<uint32_t>(ctx, p.o_small);
    ZK_CUDA(cudaMemcpyAsync(d_enc, points, 32 * n, cudaMemcpyHostToDevice, ctx->stream));
    ZK_CUDA(cudaMemcpyAsync(at<uint8_t>(ctx, p.o_scalars), scalars, 32 * n, cudaMemcpyHostToDevice, ctx->stream));
    k_jm_read_points<<<grid(n, JT), JT, 0, ctx->stream>>>(n, d_enc, at<uint32_t>(ctx, p.o_niels), reinterpret_cast<unsigned long long *>(small + 2));
    ZK_TRY(jm_msm_run(ctx, p));
    k_jm_encode<<<1, 32, 0, ctx->stream>>>(at<uint32_t>(ctx, p.o_R) + (size_t)JM_EXT_WORDS * p.W, small + 8);
    ZK_CUDA(cudaGetLastError());
    uint32_t h[16];
    ZK_CUDA(cudaMemcpyAsync(h, small, 64, cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    const unsigned long long bad = (unsigned long long)h[2] | ((unsigned long long)h[3] << 32);
    if (bad != JM_NO_BAD) {
        zk_set_error("zk_jubjub_msm: point %llu fails Point::read", bad);
        return ZK_ERR_DECODE;
    }
    memcpy(out, h + 8, 32);
    return ZK_OK;
}

// the batch check on device inputs; message i = msgs[off[i] - base .. off[i + 1] - base)
static int rj_batch_launch(zk_ctx *ctx, size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *off, uint64_t base,
                           const uint8_t *zs, uint8_t *verdict, uint64_t *first_bad) {
    if (!n) {                                        // the reference's loop does not run: O == O
        ZK_CUDA(cudaMemsetAsync(verdict, zkrj::RJ_OK, 1, ctx->stream));
        if (first_bad) ZK_CUDA(cudaMemsetAsync(first_bad, 0, 8, ctx->stream));
        return ZK_OK;
    }
    const size_t cap = (size_t)(ctx->sm_count > 0 ? ctx->sm_count : 1) * JM_BLOCKS_PER_SM;
    const size_t blocks = grid(n, JT) < cap ? grid(n, JT) : cap;
    const JmPlan p = jm_plan(2 * n + 1, 32 * blocks);
    ZK_TRY(jm_begin(ctx, p));
    uint32_t *small = at<uint32_t>(ctx, p.o_small), *niels = at<uint32_t>(ctx, p.o_niels), *scal = at<uint32_t>(ctx, p.o_scalars),
             *part = at<uint32_t>(ctx, p.o_extra);
    unsigned long long *bad = reinterpret_cast<unsigned long long *>(small + 2);
    k_rj_batch_prep<<<(unsigned)blocks, JT, 0, ctx->stream>>>(n, vks, sigs, msgs, off, base, zs, niels, scal, part, bad);
    k_rj_batch_last<<<1, 256, 0, ctx->stream>>>(n, (uint32_t)blocks, part, niels, scal);
    ZK_TRY(jm_msm_run(ctx, p));
    k_rj_batch_verdict<<<1, 32, 0, ctx->stream>>>(at<uint32_t>(ctx, p.o_R) + (size_t)JM_EXT_WORDS * p.W, bad, n, verdict, first_bad);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_redjubjub_batch_verify_device(zk_ctx *ctx, size_t n, const uint8_t *d_vks, const uint8_t *d_sigs, const uint8_t *d_msgs,
                                                const uint64_t *d_msg_off, const uint8_t *d_zs, uint8_t *d_verdict, uint64_t *d_first_bad) {
    if (!ctx || !d_verdict || (n && (!d_vks || !d_sigs || !d_msgs || !d_msg_off || !d_zs))) {
        zk_set_error("zk_redjubjub_batch_verify_device: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (2 * n + 1 > JM_MAX_POINTS) {
        zk_set_error("zk_redjubjub_batch_verify_device: n = %zu is too large", n);
        return ZK_ERR_INVALID;
    }
    ZK_TRY(zk_use_device(ctx));
    return rj_batch_launch(ctx, n, d_vks, d_sigs, d_msgs, d_msg_off, 0, d_zs, d_verdict, d_first_bad);
}

extern "C" int zk_redjubjub_batch_verify(zk_ctx *ctx, size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs,
                                         const uint64_t *msg_off, const uint8_t *zs, uint8_t *verdict, uint64_t *first_bad) {
    if (!ctx || !verdict || (n && (!vks || !sigs || !msgs || !msg_off || !zs))) {
        zk_set_error("zk_redjubjub_batch_verify: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (2 * n + 1 > JM_MAX_POINTS) {
        zk_set_error("zk_redjubjub_batch_verify: n = %zu is too large", n);
        return ZK_ERR_INVALID;
    }
    for (size_t i = 0; i < n; i++)
        if (msg_off[i + 1] < msg_off[i]) {
            zk_set_error("zk_redjubjub_batch_verify: msg_off[%zu] = %llu > msg_off[%zu] = %llu", i, (unsigned long long)msg_off[i], i + 1,
                         (unsigned long long)msg_off[i + 1]);
            return ZK_ERR_INVALID;
        }
    for (size_t i = 0; i < n; i++)
        if (!fs_bytes_canonical(zs + 32 * i)) {
            zk_set_error("zk_redjubjub_batch_verify: z[%zu] >= r_J", i);
            return ZK_ERR_NOT_CANONICAL;
        }
    if (!n) {
        *verdict = zkrj::RJ_OK;
        if (first_bad) *first_bad = 0;
        return ZK_OK;
    }
    ZK_TRY(zk_use_device(ctx));
    const uint64_t base = msg_off[0];       // the messages go up from msgs[base]; the kernel subtracts base from each offset
    uint64_t fb = 0;                        // first_bad may be NULL; the device writes it all the same
    const uint8_t *d_zs, *d_vks, *d_sigs, *d_msgs;
    const uint64_t *d_off;
    uint8_t *d_ver;
    uint64_t *d_first;
    Stage io;
    io.in(msg_off, d_off, n + 1); io.in(zs, d_zs, 32 * n); io.in(vks, d_vks, 32 * n); io.in(sigs, d_sigs, 64 * n);
    io.in(msgs + base, d_msgs, msg_off[n] - base);
    io.out(verdict, d_ver, 1); io.out(&fb, d_first, 1);
    ZK_TRY(io.up(ctx));
    ZK_TRY(rj_batch_launch(ctx, n, d_vks, d_sigs, d_msgs, d_off, base, d_zs, d_ver, d_first));
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (first_bad) *first_bad = fb;
    return ZK_OK;
}
