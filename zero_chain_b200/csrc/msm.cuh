// Pippenger multi-scalar multiplication for sm_90a (H100), templated on the base field (Fq -> G1, Fq2 -> G2).
//
// Replaces upstream bellman 0.1.0 `multiexp` (SURVEY.md §3.2 / §8 a8; call sites in create_proof:
// H, L, A, B1, B2 — reference call site core/proofs/src/confidential.rs:149).  Same mathematical
// result (sum s_i * P_i); the schedule is GPU-first rather than bellman's per-window CPU tasks:
//
//   1. k_msm_digits     scalars (canonical FrRepr) -> signed c-bit digits, layout [window][point]
//   2. k_tile_hist      per-tile bucket histograms in SHARED MEMORY (2^(c-1) counters, no global atomics)
//      k_col_scan       per-bucket prefix over tiles;  scan -> bucket offsets
//      k_scatter        counting-sort scatter with shared-memory cursors -> entries grouped by bucket
//      (windows above 16 bits: k_tile_hist bins by the high 9 key bits over many small tiles, k_bin_scan scans the
//      tiles, k_coarse_scatter groups each chunk by bin before storing it, k_fine_sort finishes each bin by the low bits)
//   3. k_accumulate     one thread per <= TASK_LEN entries of one bucket: gathers affine bases from HBM
//                       (software-prefetched), mixed additions into an XYZZ accumulator in registers
//      k_combine_*      fold the bucket's task partials (thread per bucket; warp per heavy bucket)
//   4. k_bit_sums / k_sum_points / k_finish_bits   sum_d d*B[d] as sum_b 2^b (sum of buckets with bit b of d set)
//
// "Window sets" (ws) are independent sort/bucket domains: a single MSM over precomputed tables
// 2^(c*w) * P_i uses ONE ws for all windows (no doubling tail, 2^(c-1) buckets in total); a batch of
// proofs uses one ws per proof; an ad-hoc MSM without tables uses one ws per window and finishes
// with a Horner combine.  An entry's payload is always its position inside the ws ([w][i] order),
// which is also its index into the base table.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "curve.cuh"
#include "curve_coop.cuh"
#include "msm_accum.cuh"
#include "tma.cuh"

namespace zkmsm {

constexpr int TILE = 131072;       // entries per tile of the one-level sort (one tile ~ one CTA of a single wave at 2^20 x 16 windows)
constexpr int SORT_THREADS = 1024;
// Coarse level of the two-level sort: 256-thread blocks, tiles sized so that the grid is at least two full waves of
// them (coarse_tile_len)
constexpr int COARSE_THREADS = 256;
constexpr uint32_t DIGIT_ZERO = 0xffffffffu;

// ---- 1. digits ---------------------------------------------------------------------------------
// scalars: [n_ws][n][8] canonical u32 words (value < r); digits: [n_ws][W][n].
// Signed digits d_w in (-2^(c-1), 2^(c-1)], sum d_w 2^(c w) = scalar.  Code: (|d|-1) | sign<<31, or DIGIT_ZERO.
static __global__ void k_msm_digits(const uint32_t *__restrict__ scalars, uint32_t n, int c, int W,
                             uint32_t *__restrict__ digits, int *__restrict__ err) {
    // stage this block's tile of scalars (blockDim.x * 32 B, contiguous) in shared memory with one bulk
    // asynchronous copy (TMA engine, mbarrier completion), then every thread reads its own 32 bytes
    __shared__ __align__(128) uint4 tile[256 * 2];
    __shared__ uint64_t bar;
    uint32_t i0 = blockIdx.x * blockDim.x, i = i0 + threadIdx.x;
    uint32_t ws = blockIdx.y;
    uint32_t cnt = n - i0 < blockDim.x ? n - i0 : blockDim.x;
    if (threadIdx.x == 0) zktma::mbar_init(&bar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        zktma::mbar_expect_tx(&bar, cnt * 32u);
        zktma::bulk_load(tile, scalars + ((size_t)ws * n + i0) * 8, cnt * 32u, &bar);
    }
    zktma::mbar_wait(&bar, 0);
    if (i >= n) return;
    uint4 lo = tile[2 * threadIdx.x], hi = tile[2 * threadIdx.x + 1];
    uint32_t k[9] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w, 0};
    {   // canonical check: k < r  (Fr::from_repr rejects otherwise, fr.rs:280-289)
        Fr t; for (int j = 0; j < 8; j++) t.l[j] = k[j];
        if (!Fr::canonical_lt_mod(t)) atomicExch(err, 1);
    }
    uint32_t carry = 0;
    const uint32_t half = 1u << (c - 1), full = 1u << c, mask = full - 1;
    uint32_t *out = digits + (size_t)ws * W * n + i;
    for (int w = 0; w < W; w++) {
        int bit = w * c, word = bit >> 5, sh = bit & 31;
        uint32_t v = 0;
        if (word < 8) {
            uint64_t two = (uint64_t)k[word] | ((uint64_t)k[word + 1] << 32);
            v = (uint32_t)(two >> sh) & mask;
        }
        v += carry;
        uint32_t code;
        if (v > half) { code = (full - v - 1) | 0x80000000u; carry = 1; }
        else { code = v ? (v - 1) : DIGIT_ZERO; carry = 0; }
        out[(size_t)w * n] = code;
    }
}

// ---- 2. counting sort --------------------------------------------------------------------------
// Block-wide walk over cnt consecutive elements of s (aligned to sizeof(T)): f(element, index) for every element, with
// 16-byte loads (4 digit codes or 2 {entry, key} pairs), U of them issued per thread before any is used, so that each
// thread keeps U x 16 bytes in flight.  The few elements before the first 16-byte boundary and after the last one are
// read one by one.  The order in which f sees the elements is unspecified.
template <class T, int U, class Fn>
__device__ __forceinline__ void block_for_each(const T *__restrict__ s, uint64_t cnt, Fn f) {
    static_assert(sizeof(T) == 4 || sizeof(T) == 8, "4- or 8-byte elements");
    constexpr int V = 16 / (int)sizeof(T);
    uint64_t head = ((16u - ((uint32_t)(uintptr_t)s & 15u)) & 15u) / sizeof(T);
    if (head > cnt) head = cnt;
    const uint64_t nvec = (cnt - head) / V, tail = head + nvec * V;
    if (threadIdx.x < head) f(s[threadIdx.x], (uint64_t)threadIdx.x);
    if (threadIdx.x < cnt - tail) f(s[tail + threadIdx.x], tail + threadIdx.x);
    const uint4 *v = reinterpret_cast<const uint4 *>(s + head);
    const uint64_t step = blockDim.x;
    for (uint64_t q = threadIdx.x; q < nvec; q += U * step) {
        uint4 x[U];
#pragma unroll
        for (int k = 0; k < U; k++) if (q + k * step < nvec) x[k] = __ldg(v + q + k * step);
#pragma unroll
        for (int k = 0; k < U; k++) {
            if (q + k * step >= nvec) break;
            const uint64_t i = head + (q + k * step) * V;
            if constexpr (sizeof(T) == 4) { f(x[k].x, i); f(x[k].y, i + 1); f(x[k].z, i + 2); f(x[k].w, i + 3); }
            else { f(make_uint2(x[k].x, x[k].y), i); f(make_uint2(x[k].z, x[k].w), i + 1); }
        }
    }
}
// Sort tiles: tile t of a domain holds its entries [t tile_len, (t+1) tile_len).  The per-tile counters of a domain are
// stored tile-major ([tile][bin], one-level sort: few tiles, many bins, scanned by k_col_scan) or bin-major ([bin][tile],
// coarse level: many tiles, 512 bins, scanned by k_bin_scan).
__device__ __forceinline__ size_t tile_bin_index(int ws, int tile, int b, int tiles_per_ws, int nbins, bool bin_major) {
    return bin_major ? ((size_t)ws * nbins + b) * tiles_per_ws + tile : ((size_t)ws * tiles_per_ws + tile) * nbins + b;
}
// Entries per coarse tile: the largest multiple of COARSE_CHUNK (4096) that still gives at least two waves of `resident`
// k_coarse_scatter blocks over all domains (at least one chunk).
constexpr int COARSE_PER_THREAD = 16, COARSE_CHUNK = COARSE_THREADS * COARSE_PER_THREAD;
inline uint32_t coarse_tile_len(uint64_t e_dom, size_t n_dom, int resident) {
    uint64_t t = e_dom * n_dom / (2 * (uint64_t)(resident > 0 ? resident : 1)) / COARSE_CHUNK * COARSE_CHUNK;
    return (uint32_t)(t < (uint64_t)COARSE_CHUNK ? COARSE_CHUNK : t);
}
// `shift` > 0 bins by the high bits of the bucket key (coarse level of the two-level sort used for windows above 16 bits)
static __global__ void __launch_bounds__(SORT_THREADS) k_tile_hist(const uint32_t *__restrict__ digits, uint64_t e_ws, int nbins, int shift,
                                                            uint32_t *__restrict__ tile_hist, int tiles_per_ws, uint32_t tile_len, bool bin_major) {
    extern __shared__ uint32_t sh[];
    int tile = blockIdx.x, ws = blockIdx.y;
    for (int b = threadIdx.x; b < nbins; b += blockDim.x) sh[b] = 0;
    __syncthreads();
    uint64_t p0 = (uint64_t)tile * tile_len, p1 = p0 + tile_len < e_ws ? p0 + tile_len : e_ws;
    block_for_each<uint32_t, 4>(digits + (size_t)ws * e_ws + p0, p1 - p0, [&](uint32_t code, uint64_t) {
        if (code != DIGIT_ZERO) atomicAdd(&sh[(code & 0x7fffffffu) >> shift], 1u);
    });
    __syncthreads();
    for (int b = threadIdx.x; b < nbins; b += blockDim.x) tile_hist[tile_bin_index(ws, tile, b, tiles_per_ws, nbins, bin_major)] = sh[b];
}
// thread per (ws, bin): exclusive prefix over tiles -> tile_off, total -> sizes
static __global__ void k_col_scan(const uint32_t *__restrict__ tile_hist, uint32_t *__restrict__ tile_off, uint32_t *__restrict__ sizes,
                           int nbins, int tiles_per_ws, int n_ws) {
    int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nbins * n_ws) return;
    int ws = g / nbins, b = g - ws * nbins;
    uint32_t run = 0;
    for (int t = 0; t < tiles_per_ws; t++) {
        size_t idx = ((size_t)ws * tiles_per_ws + t) * nbins + b;
        uint32_t v = tile_hist[idx];
        tile_off[idx] = run;
        run += v;
    }
    sizes[g] = run;
}
// Coarse level (bin-major counters): block per (ws, bin), exclusive prefix of the bin's counters over the tiles ->
// tile_off (same layout), total -> sizes.  The block scans COARSE_THREADS x 4 counters per step with warp shuffles.
static __global__ void __launch_bounds__(COARSE_THREADS) k_bin_scan(const uint32_t *__restrict__ tile_hist, uint32_t *__restrict__ tile_off,
                                                                    uint32_t *__restrict__ sizes, int tiles_per_ws) {
    __shared__ uint32_t wsum[COARSE_THREADS / 32];
    const uint32_t *in = tile_hist + (size_t)blockIdx.x * tiles_per_ws;
    uint32_t *out = tile_off + (size_t)blockIdx.x * tiles_per_ws;
    uint32_t run = 0;
    for (int base = 0; base < tiles_per_ws; base += COARSE_THREADS * 4) {
        const int t0 = base + threadIdx.x * 4;
        uint32_t v[4], s = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) { v[k] = t0 + k < tiles_per_ws ? in[t0 + k] : 0; s += v[k]; }
        uint32_t inc = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= (unsigned)o) inc += t; }
        if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = inc;
        __syncthreads();
        uint32_t before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < COARSE_THREADS / 32; w++) { const uint32_t x = wsum[w]; before += w < (int)(threadIdx.x >> 5) ? x : 0; total += x; }
        uint32_t ex = run + before + inc - s;
#pragma unroll
        for (int k = 0; k < 4; k++) { if (t0 + k < tiles_per_ws) out[t0 + k] = ex; ex += v[k]; }
        run += total;
        __syncthreads();                               // wsum is rewritten by the next step
    }
    if (threadIdx.x == 0) sizes[blockIdx.x] = run;
}
// one-level sort: entries go straight from the digits to their bucket's cursor
static __global__ void __launch_bounds__(SORT_THREADS) k_scatter(const uint32_t *__restrict__ digits, uint64_t e_ws, int nbins,
                                                          const uint32_t *__restrict__ tile_off, const uint32_t *__restrict__ bucket_off,
                                                          uint32_t *__restrict__ sorted, int tiles_per_ws, uint32_t tile_len) {
    extern __shared__ uint32_t sh[];
    int tile = blockIdx.x, ws = blockIdx.y;
    const uint32_t *bo = bucket_off + (size_t)ws * nbins;
    for (int b = threadIdx.x; b < nbins; b += blockDim.x) sh[b] = bo[b] + tile_off[tile_bin_index(ws, tile, b, tiles_per_ws, nbins, false)];
    __syncthreads();
    uint64_t p0 = (uint64_t)tile * tile_len, p1 = p0 + tile_len < e_ws ? p0 + tile_len : e_ws;
    block_for_each<uint32_t, 4>(digits + (size_t)ws * e_ws + p0, p1 - p0, [&](uint32_t code, uint64_t i) {
        if (code != DIGIT_ZERO) sorted[atomicAdd(&sh[code & 0x7fffffffu], 1u)] = (uint32_t)(p0 + i) | (code & 0x80000000u);
    });
}
// Coarse level of the two-level sort: each entry is stored as {payload, bucket key}, so that k_fine_sort reads the key
// with the entry instead of gathering it from the digits array (a random 4-byte read costs a 32-byte sector).  A tile is
// taken in chunks of COARSE_CHUNK entries (16 loads in flight per thread); each chunk is first grouped by coarse bin in
// shared memory, so that the global stores are runs of consecutive addresses per bin instead of one 8-byte store per
// sector (8 entries per bin and chunk on average at 512 bins).
constexpr int COARSE_BINS = 512;
static __global__ void __launch_bounds__(COARSE_THREADS) k_coarse_scatter(const uint32_t *__restrict__ digits, uint64_t e_ws, int shift,
                                                                          const uint32_t *__restrict__ tile_off, const uint32_t *__restrict__ bin_off,
                                                                          uint2 *__restrict__ sorted, int tiles_per_ws, uint32_t tile_len) {
    __shared__ uint2 stage[COARSE_CHUNK];
    __shared__ uint32_t cur[COARSE_BINS], cnt[COARSE_BINS], loff[COARSE_BINS], wsum[COARSE_THREADS / 32 + 1];
    const int tile = blockIdx.x, ws = blockIdx.y;
    for (int b = threadIdx.x; b < COARSE_BINS; b += COARSE_THREADS)
        cur[b] = bin_off[(size_t)ws * COARSE_BINS + b] + tile_off[tile_bin_index(ws, tile, b, tiles_per_ws, COARSE_BINS, true)];
    const uint64_t p0 = (uint64_t)tile * tile_len, p1 = p0 + tile_len < e_ws ? p0 + tile_len : e_ws;
    const uint32_t *d = digits + (size_t)ws * e_ws;
    for (uint64_t c0 = p0; c0 < p1; c0 += COARSE_CHUNK) {
        for (int b = threadIdx.x; b < COARSE_BINS; b += COARSE_THREADS) cnt[b] = 0;
        __syncthreads();
        uint32_t code[COARSE_PER_THREAD], rank[COARSE_PER_THREAD];
#pragma unroll
        for (int k = 0; k < COARSE_PER_THREAD; k++) {
            const uint64_t p = c0 + threadIdx.x + k * COARSE_THREADS;
            code[k] = p < p1 ? __ldg(d + p) : DIGIT_ZERO;
        }
#pragma unroll
        for (int k = 0; k < COARSE_PER_THREAD; k++)
            if (code[k] != DIGIT_ZERO) rank[k] = atomicAdd(&cnt[(code[k] & 0x7fffffffu) >> shift], 1u);
        __syncthreads();
        {   // exclusive scan of the 512 chunk counters, two per thread
            const uint32_t a = cnt[2 * threadIdx.x], b = cnt[2 * threadIdx.x + 1], s = a + b;
            uint32_t inc = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= (unsigned)o) inc += t; }
            if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = inc;
            __syncthreads();
            uint32_t before = 0;
            for (int w = 0; w < (int)(threadIdx.x >> 5); w++) before += wsum[w];
            const uint32_t ex = before + inc - s;
            loff[2 * threadIdx.x] = ex;
            loff[2 * threadIdx.x + 1] = ex + a;
            if (threadIdx.x == COARSE_THREADS - 1) wsum[COARSE_THREADS / 32] = ex + s;     // entries of the chunk
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < COARSE_PER_THREAD; k++)
            if (code[k] != DIGIT_ZERO) {
                const uint32_t key = code[k] & 0x7fffffffu;
                const uint32_t entry = (uint32_t)(c0 + threadIdx.x + k * COARSE_THREADS) | (code[k] & 0x80000000u);
                stage[loff[key >> shift] + rank[k]] = make_uint2(entry, key);
            }
        __syncthreads();
        const uint32_t total = wsum[COARSE_THREADS / 32];
        for (uint32_t j = threadIdx.x; j < total; j += COARSE_THREADS) {
            const uint2 e = stage[j];
            const uint32_t b = e.y >> shift;
            sorted[cur[b] + j - loff[b]] = e;
        }
        __syncthreads();
        for (int b = threadIdx.x; b < COARSE_BINS; b += COARSE_THREADS) cur[b] += cnt[b];
    }
}

// Fine level of the two-level sort (windows above 16 bits: 2^(c-1) buckets no longer fit a shared-memory histogram).
// One block per (coarse bin, domain): the entries of the coarse bin (already contiguous) are counted by the low `low`
// bits of their key in shared memory, the counts are scanned, and the entries are scattered to their final places.
// Writes bucket sizes and bucket offsets directly (no global scan needed); the bucket key of an entry comes with it from
// k_coarse_scatter, so every pass reads the coarse bin contiguously, with 16-byte loads of two entries and four loads in
// flight per thread.
// The scatter goes to a FINE_STAGE-entry window of shared memory that is then copied out with coalesced stores: one
// 4-byte store per entry straight to HBM would leave hundreds of blocks' whole output regions as partly written sectors in
// L2 at once.  A bin whose output is larger than the window is scattered in segments of consecutive buckets that fit it,
// one more pass over the bin per segment; a bucket larger than the window, or a bin of more than FINE_MAX_SEGMENTS
// windows, is scattered straight to HBM instead.
constexpr int FINE_STAGE = 25 * 1024, FINE_MAX_SEGMENTS = 4;      // 100 KB of shared memory: two blocks per SM
static __global__ void __launch_bounds__(1024, 2) k_fine_sort(const uint2 *__restrict__ coarse_sorted, const uint32_t *__restrict__ coarse_off,
                                                          int n_coarse, int low,
                                                          uint32_t *__restrict__ sizes, uint32_t *__restrict__ bucket_off, uint32_t *__restrict__ sorted) {
    extern __shared__ uint32_t stage[];                  // FINE_STAGE entries
    __shared__ uint32_t hist[1024], off[1025];
    __shared__ uint32_t wsum[32];
    const int cb = blockIdx.x, dom = blockIdx.y, g = dom * n_coarse + cb;
    const uint32_t r0 = coarse_off[g], r1 = coarse_off[g + 1], nb = 1u << low, fmask = nb - 1u;
    hist[threadIdx.x] = 0;
    __syncthreads();
    block_for_each<uint2, 4>(coarse_sorted + r0, r1 - r0, [&](uint2 e, uint64_t) { atomicAdd(&hist[e.y & fmask], 1u); });
    __syncthreads();
    // exclusive scan of the (<= 1024) counters: one per thread
    uint32_t v = threadIdx.x < nb ? hist[threadIdx.x] : 0, inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= (unsigned)o) inc += t; }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = inc;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint32_t w = wsum[threadIdx.x], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, wi, o); if (threadIdx.x >= (unsigned)o) wi += t; }
        wsum[threadIdx.x] = wi - w;
    }
    __syncthreads();
    uint32_t excl = inc - v + wsum[threadIdx.x >> 5];
    __syncthreads();
    if (threadIdx.x < nb) {
        size_t b = ((size_t)g << low) + threadIdx.x;
        sizes[b] = v;
        bucket_off[b] = r0 + excl;
        hist[threadIdx.x] = r0 + excl;           // becomes the scatter cursor
        off[threadIdx.x] = excl;                 // bucket start inside the bin
        if (threadIdx.x == nb - 1) off[nb] = excl + v;
    }
    if (cb == n_coarse - 1 && dom == (int)gridDim.y - 1 && threadIdx.x == 0) bucket_off[((size_t)g + 1) << low] = r1;
    __syncthreads();
    const uint32_t total = r1 - r0;
    if (total > (uint32_t)FINE_MAX_SEGMENTS * FINE_STAGE) {
        block_for_each<uint2, 4>(coarse_sorted + r0, total, [&](uint2 e, uint64_t) { sorted[atomicAdd(&hist[e.y & fmask], 1u)] = e.x; });
        return;
    }
    for (uint32_t lo = 0; lo < nb;) {                    // segment [lo, hi) of buckets, the same on every thread
        const uint32_t base = off[lo];
        const int fit = __syncthreads_count(threadIdx.x >= lo && threadIdx.x < nb && off[threadIdx.x + 1] - base <= (uint32_t)FINE_STAGE);
        const uint32_t hi = lo + (fit > 0 ? (uint32_t)fit : 1u);
        const bool direct = fit == 0;                    // bucket lo alone is larger than the window
        block_for_each<uint2, 2>(coarse_sorted + r0, total, [&](uint2 e, uint64_t) {     // 2 loads in flight: 32 registers
            const uint32_t k = e.y & fmask;
            if (k >= lo && k < hi) {
                const uint32_t p = atomicAdd(&hist[k], 1u);
                if (direct) sorted[p] = e.x;
                else stage[p - r0 - base] = e.x;
            }
        });
        __syncthreads();
        if (!direct)
            for (uint32_t j = threadIdx.x, m = off[hi] - base; j < m; j += blockDim.x) sorted[r0 + base + j] = stage[j];
        __syncthreads();
        lo = hi;
    }
}

// ---- generic exclusive scan of u32 (three-phase; out[n] = total) -----------------------------------
constexpr int SCAN_T = 256, SCAN_E = 8, SCAN_B = SCAN_T * SCAN_E;
// number of tasks of a bucket with v entries for task length L: round to nearest (at least one), so that the
// task count tracks total/L instead of overshooting by half a task per bucket (k_accumulate splits evenly)
template <bool TASKS>
__device__ __forceinline__ uint32_t scan_load(const uint32_t *in, size_t i, uint32_t task_len) {
    uint32_t v = in[i];
    if (!TASKS) return v;
    if (v == 0) return 0;
    uint32_t t = (v + task_len / 2) / task_len;
    return t ? t : 1;
}
// Task length from the number of non-zero entries (bucket_off[NB]).  Tasks all take the same time, so the
// accumulation kernel runs in waves of `capacity` (= resident threads) tasks; the length is chosen so that the
// task count is just under a whole number of waves (a trailing partial wave costs a full wave's latency).
static __global__ void k_pick_task_len(const uint32_t *__restrict__ total_entries, const uint32_t *__restrict__ sorted_entries, uint32_t *__restrict__ task_len,
                                       uint32_t capacity, unsigned long long *__restrict__ work_counter, unsigned long long *__restrict__ xyzz_counter) {
    task_len[1] = 0;                                           // heavy-bucket counter of k_combine_serial (next word)
    uint32_t total = *total_entries;                           // entries the XYZZ pass sees (after the batched-affine rounds)
    *work_counter += *sorted_entries;                          // all bucket additions of this MSM (non-zero digits)
    *xyzz_counter += total;                                    // ... of which this many are left to the XYZZ pass                                    // executed bucket additions (non-zero digits) of this context, read by zk_ctx_profile_counts
    uint32_t waves = (total + (uint32_t)TASK_LEN_MAX * capacity - 1) / ((uint32_t)TASK_LEN_MAX * capacity);
    if (waves < 2) waves = 2;                                   // small inputs: at least two waves of short tasks
    uint32_t target = (uint32_t)(0.97f * (float)waves * (float)capacity);
    uint32_t t = (total + target - 1) / (target ? target : 1);
    if (t < (uint32_t)TASK_LEN_MIN) t = TASK_LEN_MIN;
    if (t > (uint32_t)TASK_LEN_MAX + 8) t = TASK_LEN_MAX + 8;
    *task_len = t;
}
// TASKS: scan ceil(in / *task_len_p) instead of in
template <bool TASKS>
__global__ void __launch_bounds__(SCAN_T) k_scan_block(const uint32_t *__restrict__ in, uint32_t *__restrict__ out,
                                                       uint32_t *__restrict__ block_sums, size_t n, const uint32_t *__restrict__ task_len_p) {
    __shared__ uint32_t wsum[SCAN_T / 32];
    const uint32_t task_len = TASKS ? *task_len_p : 1u;
    size_t base = (size_t)blockIdx.x * SCAN_B + (size_t)threadIdx.x * SCAN_E;
    uint32_t v[SCAN_E], s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_E; k++) { v[k] = base + k < n ? scan_load<TASKS>(in, base + k, task_len) : 0; s += v[k]; }
    uint32_t inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= o) inc += t; }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = inc;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint32_t w = threadIdx.x < SCAN_T / 32 ? wsum[threadIdx.x] : 0, wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, wi, o); if (threadIdx.x >= o) wi += t; }
        if (threadIdx.x < SCAN_T / 32) wsum[threadIdx.x] = wi - w;
        if (threadIdx.x == SCAN_T / 32 - 1 && block_sums) block_sums[blockIdx.x] = wi;
    }
    __syncthreads();
    uint32_t ex = inc - s + wsum[threadIdx.x >> 5];
#pragma unroll
    for (int k = 0; k < SCAN_E; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
}
static __global__ void k_scan_add(uint32_t *__restrict__ out, const uint32_t *__restrict__ block_off, size_t n) {
    size_t i = (size_t)blockIdx.x * SCAN_B + threadIdx.x;
    uint32_t o = block_off[blockIdx.x];
    for (int k = 0; k < SCAN_E; k++, i += SCAN_T) if (i < n) out[i] += o;
}
// out[0..n) = exclusive prefix sums of in (or of ceil(in / *task_len_p) when TASKS), out[n] = total.
// scratch must hold >= 2 * (n / SCAN_B + 8) words.
template <bool TASKS>
inline void exclusive_scan(const uint32_t *in, uint32_t *out, size_t n, uint32_t *scratch, cudaStream_t st, const uint32_t *task_len_p = nullptr) {
    size_t nb = (n + SCAN_B - 1) / SCAN_B;
    if (nb == 0) nb = 1;
    uint32_t *bs = scratch;
    k_scan_block<TASKS><<<(unsigned)nb, SCAN_T, 0, st>>>(in, out, bs, n, task_len_p);
    if (nb == 1) {
        cudaMemcpyAsync(out + n, bs, 4, cudaMemcpyDeviceToDevice, st);
        return;
    }
    uint32_t *bo = scratch + nb + 1;
    exclusive_scan<false>(bs, bo, nb, bo + nb + 2, st);          // bo[nb] = grand total
    k_scan_add<<<(unsigned)nb, SCAN_T, 0, st>>>(out, bo, n);
    cudaMemcpyAsync(out + n, bo + nb, 4, cudaMemcpyDeviceToDevice, st);
}

// ---- 2c. task order by length -------------------------------------------------------------------------------------
// Tasks of one warp should run the same number of additions.  With ~equal buckets (one big MSM, 16-bit windows) they do;
// with short Poisson-distributed buckets (batched proving, wide windows) they do not, and a warp runs as long as its
// longest task.  Tasks are therefore issued in order of DECREASING length: a counting sort of the tasks by length
// (<= 255 after clamping), block-aggregated so that global atomics are one per (block, length).
constexpr int LEN_BINS = 256, LEN_BLOCK = 1024;
__device__ __forceinline__ uint32_t task_len_of(const uint32_t *bucket_off, const uint32_t *task_off, uint32_t b, uint32_t &nt) {
    nt = task_off[b + 1] - task_off[b];
    if (!nt) return 0;
    uint32_t size = bucket_off[b + 1] - bucket_off[b], len = (size + nt - 1) / nt;
    return len < (uint32_t)LEN_BINS ? len : (uint32_t)LEN_BINS - 1;
}
static __global__ void __launch_bounds__(LEN_BLOCK) k_len_hist(const uint32_t *__restrict__ bucket_off, const uint32_t *__restrict__ task_off,
                                                              uint32_t n_buckets, uint32_t *__restrict__ ghist) {
    __shared__ uint32_t sh[LEN_BINS];
    if (threadIdx.x < LEN_BINS) sh[threadIdx.x] = 0;
    __syncthreads();
    uint32_t b = blockIdx.x * LEN_BLOCK + threadIdx.x, nt = 0;
    if (b < n_buckets) { uint32_t len = task_len_of(bucket_off, task_off, b, nt); if (nt) atomicAdd(&sh[len], nt); }
    __syncthreads();
    if (threadIdx.x < LEN_BINS && sh[threadIdx.x]) atomicAdd(&ghist[threadIdx.x], sh[threadIdx.x]);
}
// one block: cursor[l] = number of tasks longer than l (exclusive scan from the long end); ghist is cleared for the next MSM
static __global__ void __launch_bounds__(LEN_BINS) k_len_scan(uint32_t *__restrict__ ghist, uint32_t *__restrict__ cursor) {
    __shared__ uint32_t sh[LEN_BINS];
    sh[threadIdx.x] = ghist[LEN_BINS - 1 - threadIdx.x];      // reversed: index 0 = longest
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t run = 0; for (int i = 0; i < LEN_BINS; i++) { uint32_t v = sh[i]; sh[i] = run; run += v; } }
    __syncthreads();
    cursor[LEN_BINS - 1 - threadIdx.x] = sh[threadIdx.x];
    ghist[threadIdx.x] = 0;
}
static __global__ void __launch_bounds__(LEN_BLOCK) k_len_place(const uint32_t *__restrict__ bucket_off, const uint32_t *__restrict__ task_off,
                                                               uint32_t n_buckets, uint32_t *__restrict__ cursor, uint32_t *__restrict__ order) {
    __shared__ uint32_t cnt[LEN_BINS], base[LEN_BINS];
    if (threadIdx.x < LEN_BINS) cnt[threadIdx.x] = 0;
    __syncthreads();
    uint32_t b = blockIdx.x * LEN_BLOCK + threadIdx.x, nt = 0, len = 0, local = 0;
    if (b < n_buckets) { len = task_len_of(bucket_off, task_off, b, nt); if (nt) local = atomicAdd(&cnt[len], nt); }
    __syncthreads();
    if (threadIdx.x < LEN_BINS && cnt[threadIdx.x]) base[threadIdx.x] = atomicAdd(&cursor[threadIdx.x], cnt[threadIdx.x]);
    __syncthreads();
    if (nt) {
        uint32_t pos = base[len] + local, t0 = task_off[b];
        for (uint32_t s = 0; s < nt; s++) order[pos + s] = t0 + s;
    }
}

// ---- 3. bucket accumulation: k_accumulate lives in msm_accum.cuh (shared with the hot translation unit) ----
// buckets[b] = sum of the bucket's task partials.  Thread per bucket for the common short case (serial
// adds; a warp with few live lanes wastes its issue slots), one warp per bucket for heavy (skewed) buckets.
constexpr uint32_t COMB_SERIAL_MAX = 32;
template <class F>
__global__ void __launch_bounds__(128) k_combine_serial(const XYZZ<F> *__restrict__ partials, const uint32_t *__restrict__ task_off,
                                                        uint32_t n_buckets, XYZZ<F> *__restrict__ buckets,
                                                        uint32_t *__restrict__ heavy_list, uint32_t *__restrict__ heavy_count) {
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_buckets) return;
    uint32_t t0 = task_off[b], t1 = task_off[b + 1];
    if (t1 - t0 > COMB_SERIAL_MAX) { heavy_list[atomicAdd(heavy_count, 1u)] = b; return; }     // rare: left to k_combine_warp
    XYZZ<F> acc = XYZZ<F>::inf();
    if (t1 > t0) acc = partials[t0];
    for (uint32_t t = t0 + 1; t < t1; t++) acc.add(partials[t]);
    buckets[b] = acc;
}
// fixed-size grid: warp w folds the heavy buckets heavy_list[w], heavy_list[w + n_warps], ...
template <class F>
__global__ void __launch_bounds__(128) k_combine_warp(const XYZZ<F> *__restrict__ partials, const uint32_t *__restrict__ task_off,
                                                      const uint32_t *__restrict__ heavy_list, const uint32_t *__restrict__ heavy_count,
                                                      XYZZ<F> *__restrict__ buckets) {
    extern __shared__ unsigned char smraw[];
    XYZZ<F> *sm = reinterpret_cast<XYZZ<F> *>(smraw) + (threadIdx.x >> 5) * 32;
    const uint32_t lane = threadIdx.x & 31, n_warps = (gridDim.x * blockDim.x) >> 5, n_heavy = *heavy_count;
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_heavy; i += n_warps) {
        uint32_t b = heavy_list[i], t0 = task_off[b], t1 = task_off[b + 1];
        XYZZ<F> acc = XYZZ<F>::inf();
        for (uint32_t t = t0 + lane; t < t1; t += 32) acc.add(partials[t]);
        __syncwarp();
        sm[lane] = acc;
        __syncwarp();
        for (int o = 16; o > 0; o >>= 1) {
            if (lane < (uint32_t)o) { XYZZ<F> x = sm[lane]; x.add(sm[lane + o]); sm[lane] = x; }
            __syncwarp();
        }
        if (lane == 0) buckets[b] = sm[0];
    }
}

// ---- 4. bucket reduction: R = sum_{d=1..N} d * B[d-1] ------------------------------------------------
// Serial point additions are slow on a GPU thread (a long dependent chain each), so the reduction is organised for
// DEPTH, not work: R = sum_b 2^b X_b with X_b = sum of the buckets whose digit value d has bit b set.
// The X_b are plain sums (parallel trees, two stages), followed by one short Horner chain per domain.
//   stage 1: block (slice, bit, dom) -> partial sum of the qualifying buckets of its slice
//   stage 2: k_sum_points over the slice partials -> X[dom][bit]
//   stage 3: k_finish_bits: thread per dom, R = X_0 + 2 (X_1 + 2 (X_2 + ...))
constexpr int RED_T = 128, RED_SLICE = 512;
#ifndef ZK_RC_GL
#define ZK_RC_GL 8        // lanes per row / column of the batched-domain bucket reduction
#endif
constexpr int RC_GL = ZK_RC_GL;
#ifndef ZK_RC_MINB
#define ZK_RC_MINB 2      // resident blocks per SM of the G1 row/column sums (register budget 255 / 168 / 128)
#endif
// warp-level tree over the 32 lane accumulators of one warp (slot = this warp's 32 shared-memory points)
template <class F>
__device__ __forceinline__ void warp_tree(XYZZ<F> *slot, XYZZ<F> &acc, uint32_t lane) {
    slot[lane] = acc;
    __syncwarp();
    for (int o = 16; o > 0; o >>= 1) {
        if (lane < o) { XYZZ<F> x = slot[lane]; x.add(slot[lane + o]); slot[lane] = x; }
        __syncwarp();
    }
    acc = slot[0];
}
// one WARP per (slice, bit, dom): lanes stride over the slice's buckets, then a 5-level tree
template <class F>
__global__ void __launch_bounds__(RED_T) k_bit_sums(const XYZZ<F> *__restrict__ B, int N, int n_slices, int n_bits, int n_dom,
                                                    XYZZ<F> *__restrict__ part) {
    extern __shared__ unsigned char smraw[];
    uint32_t lane = threadIdx.x & 31;
    XYZZ<F> *slot = reinterpret_cast<XYZZ<F> *>(smraw) + (threadIdx.x >> 5) * 32;
    size_t gw = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (gw >= (size_t)n_slices * n_bits * n_dom) return;
    int slice = (int)(gw % n_slices), bit = (int)((gw / n_slices) % n_bits), dom = (int)(gw / ((size_t)n_slices * n_bits));
    const XYZZ<F> *p = B + (size_t)dom * N;
    // the k-th digit value d in [1, N] with bit `bit` set: d = ((k >> bit) << (bit + 1)) | 1 << bit | (k & (2^bit - 1)).
    // Lanes stride over k, so there is no divergence on the bit test; a slice is RED_SLICE/2 consecutive k.
    uint32_t k0 = (uint32_t)slice * (RED_SLICE / 2), k1 = k0 + RED_SLICE / 2;
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t k = k0 + lane; k < k1; k += 32) {
        uint32_t d = ((k >> bit) << (bit + 1)) | (1u << bit) | (k & ((1u << bit) - 1u));
        if (d <= (uint32_t)N) acc.add(p[d - 1]);
    }
    warp_tree(slot, acc, lane);
    if (lane == 0) part[((size_t)dom * n_bits + bit) * n_slices + slice] = acc;
}
// one WARP per group: out[g] = sum_{j<N} P[g*N + j]
template <class F>
__global__ void __launch_bounds__(RED_T) k_sum_points(const XYZZ<F> *__restrict__ P, int N, int n_groups, XYZZ<F> *__restrict__ out) {
    extern __shared__ unsigned char smraw[];
    uint32_t lane = threadIdx.x & 31;
    XYZZ<F> *slot = reinterpret_cast<XYZZ<F> *>(smraw) + (threadIdx.x >> 5) * 32;
    size_t g = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (g >= (size_t)n_groups) return;
    const XYZZ<F> *p = P + g * N;
    XYZZ<F> acc = XYZZ<F>::inf();
    for (int j = lane; j < N; j += 32) acc.add(p[j]);
    warp_tree(slot, acc, lane);
    if (lane == 0) out[g] = acc;
}
// one BLOCK per domain: R = sum_b 2^b X_b as a binary tree — at level s the pair (i, i + 2^s), i % 2^(s+1) == 0, becomes
// X_i += 2^(2^s) * X_(i+2^s).  Serial depth 15 doublings + 4 additions (n_bits <= 16) instead of 15 + 15 for a Horner chain, and every
// pair of a level has its own WARP running the doublings / the addition cooperatively (curve_coop.cuh: 3 / 4 dependent stages instead
// of 9 / 14 products), which is what matters here: the kernel is pure latency (one domain for a single MSM).
constexpr int FIN_WARPS = 10;          // pairs of the first level: n_bits <= 20
template <class F>
__global__ void __launch_bounds__(FIN_WARPS * 32) k_finish_bits(const XYZZ<F> *__restrict__ X, int n_bits, int n_dom, XYZZ<F> *__restrict__ R) {
    extern __shared__ unsigned char smraw[];
    XYZZ<F> *vals = reinterpret_cast<XYZZ<F> *>(smraw);          // 2 * FIN_WARPS points
    const int dom = blockIdx.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (dom >= n_dom) return;
    if (threadIdx.x < 2 * FIN_WARPS) vals[threadIdx.x] = (int)threadIdx.x < n_bits ? X[(size_t)dom * n_bits + threadIdx.x] : XYZZ<F>::inf();
    __syncthreads();
    for (int s = 0; (1 << s) < n_bits; s++) {
        const int step = 1 << s, i = w * 2 * step;
        if (i + step < n_bits) {                                 // warp-uniform
            XYZZ<F> hi = vals[i + step], v = vals[i];
            for (int k = 0; k < step; k++) zkcoop::dbl(hi);
            zkcoop::add(v, hi);
            __syncwarp();                                        // every lane has read vals[i] before lane 0 overwrites it
            if (lane == 0) vals[i] = v;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) R[dom] = vals[0];
}
// ---- two-level bucket reduction for many domains (batched proving) -----------------------------------------
// sum_d d*B[d] with d = hi*S + lo (S = 2^s):  S * sum_hi hi*R_hi + sum_lo lo*C_lo,  R_hi / C_lo = row / column sums
// of the bucket matrix.  Every bucket is added twice (instead of ~c/2 times by the per-bit subset sums); the two small
// weighted sums that remain go through the per-bit kernels above.  Used when there are enough domains to fill the GPU
// (work-bound regime); a single large MSM keeps the shallower per-bit scheme (latency-bound regime).
// EIGHT lanes per (domain, row hi = 1..N/S) or (domain, column lo = 1..S-1): each lane adds every 8th element serially,
// then a 3-level tree inside the group (a full warp per row would spend most of its issue slots in the tree).
// rows[dom][hi-1], cols[dom][lo-1].
// Output rc[(2*dom + which) * NR + idx], NR = N >> s: which = 0 rows (idx = hi-1), which = 1 columns (idx = lo-1, the
// tail idx >= S-1 stays at the all-zero infinity pattern written by a memset), so ONE per-bit reduction over 2*n_dom
// pseudo-domains of NR points finishes both weighted sums.
// GL lanes per item: 8 for many domains (work-bound), 32 inside a warp.
// one out-of-line copy of the full addition for k_rowcol_sums: inlined at its three call sites the kernel was ~21 000 instructions and
// spent more cycles waiting for instructions than issuing them
template <class F>
__device__ __noinline__ void add_outline(XYZZ<F> &acc, const XYZZ<F> &o) { acc.add(o); }
template <class F, int GL>
__global__ void __launch_bounds__(RED_T, (sizeof(F) == sizeof(Fq) ? ZK_RC_MINB : 1)) k_rowcol_sums(const XYZZ<F> *__restrict__ B, int N, int s, int n_dom, XYZZ<F> *__restrict__ rc) {
    extern __shared__ unsigned char smraw[];
    const uint32_t lane = threadIdx.x & 31, sub = lane & (GL - 1);
    XYZZ<F> *slot = reinterpret_cast<XYZZ<F> *>(smraw) + (threadIdx.x >> 5) * 32;
    const int S = 1 << s, nr = N >> s, nc = S - 1;
    const size_t n_items = (size_t)n_dom * (nr + nc);
    size_t item = ((((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * (32 / GL)) + (lane / GL);
    const bool live = item < n_items;
    int dom = 0, idx = 0;
    XYZZ<F> acc = XYZZ<F>::inf();
    if (live) {
        dom = (int)(item / (nr + nc)); idx = (int)(item % (nr + nc));
        const XYZZ<F> *p = B + (size_t)dom * N;
        if (idx < nr) {
            int hi = idx + 1;
            for (int lo = sub; lo < S; lo += GL) { int d = hi * S + lo; if (d <= N) add_outline(acc, p[d - 1]); }
        } else {
            int lo = idx - nr + 1;
            for (int hi = sub; hi <= nr; hi += GL) { int d = hi * S + lo; if (d <= N) add_outline(acc, p[d - 1]); }
        }
    }
    slot[lane] = acc;
    __syncwarp();
    for (int o = GL / 2; o > 0; o >>= 1) {
        if (sub < (uint32_t)o) { XYZZ<F> x = slot[lane]; add_outline(x, slot[lane + o]); slot[lane] = x; }
        __syncwarp();
    }
    if (live && sub == 0) {
        if (idx < nr) rc[((size_t)2 * dom) * nr + idx] = slot[lane]; else rc[((size_t)2 * dom + 1) * nr + (idx - nr)] = slot[lane];
    }
}
// A single large domain has few, long rows / columns.  Trees waste issue slots (a warp-level add costs a full warp even with
// one live lane), so the sums are done as three stages of purely SERIAL per-thread sums over short runs:
//   stage 1  thread (slot, k): elements [k*L1, (k+1)*L1) of the slot's row / column        -> t1[slot][k],  P1 partials
//   stage 2  thread (slot, k): t1[slot][k*L2 .. (k+1)*L2)                                   -> t2[slot][k],  P2 partials
//   stage 3  thread slot:      sum of t2[slot][0..P2)                                       -> rc[slot]
// Slots are enumerated in the rc layout (slot = (2*dom + which) * NR + idx); unused column slots produce infinity.
constexpr int RC_L1 = 16, RC_L2 = 8;
template <class F>
__global__ void __launch_bounds__(RED_T) k_rowcol_stage1(const XYZZ<F> *__restrict__ B, int N, int s, int n_dom, int P1, XYZZ<F> *__restrict__ t1) {
    const int S = 1 << s, nr = N >> s, nc = S - 1;
    // dense enumeration of the live (slot, run) pairs: all row runs first, then all column runs (t1 is pre-zeroed = infinity)
    const int P1r = (S + RC_L1 - 1) / RC_L1, P1c = (nr + 1 + RC_L1 - 1) / RC_L1;
    size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n_row = (size_t)n_dom * nr * P1r, n_col = (size_t)n_dom * nc * P1c;
    if (id >= n_row + n_col) return;
    int dom, idx, k, which;
    if (id < n_row) { which = 0; k = (int)(id % P1r); size_t q = id / P1r; idx = (int)(q % nr); dom = (int)(q / nr); }
    else { id -= n_row; which = 1; k = (int)(id % P1c); size_t q = id / P1c; idx = (int)(q % nc); dom = (int)(q / nc); }
    const XYZZ<F> *p = B + (size_t)dom * N;
    XYZZ<F> acc = XYZZ<F>::inf();
    if (which == 0) {
        int hi = idx + 1, lo1 = (k + 1) * RC_L1 < S ? (k + 1) * RC_L1 : S;
        for (int lo = k * RC_L1; lo < lo1; lo++) { int d = hi * S + lo; if (d <= N) acc.add(p[d - 1]); }
    } else {
        int lo = idx + 1, h1 = (k + 1) * RC_L1 < nr + 1 ? (k + 1) * RC_L1 : nr + 1;
        for (int hi = k * RC_L1; hi < h1; hi++) { int d = hi * S + lo; if (d <= N) acc.add(p[d - 1]); }
    }
    t1[((size_t)(2 * dom + which) * nr + idx) * P1 + k] = acc;
}
// out[g][k] = sum in[g][k*L .. min((k+1)*L, P_in));  P_out = ceil(P_in / L)
template <class F>
__global__ void __launch_bounds__(RED_T) k_seg_sums(const XYZZ<F> *__restrict__ in, size_t n_groups, int P_in, int L, int P_out, XYZZ<F> *__restrict__ out) {
    size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= n_groups * P_out) return;
    const size_t g = id / P_out; const int k = (int)(id % P_out);
    const XYZZ<F> *p = in + g * P_in;
    int j1 = (k + 1) * L < P_in ? (k + 1) * L : P_in;
    XYZZ<F> acc = XYZZ<F>::inf();
    for (int j = k * L; j < j1; j++) acc.add(p[j]);
    out[id] = acc;
}
// WARP per domain: R = 2^s * Rrc[2 dom] + Rrc[2 dom + 1]; the s doublings and the addition run warp-cooperatively (curve_coop.cuh)
template <class F>
__global__ void __launch_bounds__(128) k_join_rowcol(const XYZZ<F> *__restrict__ Rrc, int s, int n_dom, XYZZ<F> *__restrict__ R) {
    int dom = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (dom >= n_dom) return;
    XYZZ<F> r = Rrc[2 * dom];
    for (int k = 0; k < s; k++) zkcoop::dbl(r);
    zkcoop::add(r, Rrc[2 * dom + 1]);
    if ((threadIdx.x & 31) == 0) R[dom] = r;
}

// one WARP: out = sum_w 2^(c w) R[w]  (Horner over windows; ad-hoc MSM without tables).  The (W - 1) c doublings are inherently
// serial; each runs as three warp-cooperative stages instead of nine dependent products.
template <class F>
__global__ void __launch_bounds__(32) k_horner_windows(const XYZZ<F> *__restrict__ R, int W, int c, XYZZ<F> *__restrict__ out) {
    XYZZ<F> r = R[W - 1];
    for (int w = W - 2; w >= 0; w--) {
        for (int k = 0; k < c; k++) zkcoop::dbl(r);
        zkcoop::add(r, R[w]);
    }
    if (threadIdx.x == 0) out[0] = r;
}

// ---- precomputed tables: tbl[w][i] = 2^(c w) P_i (affine), w = 0..W-1 -------------------------------
// thread handles PRE_K points; per window: c doublings each, then one shared inversion (Montgomery trick).
constexpr int PRE_K = 4;
template <class F>
__global__ void __launch_bounds__(128) k_precompute(Affine<F> *__restrict__ tbl, uint32_t n, int c, int W) {
    uint32_t i0 = (blockIdx.x * blockDim.x + threadIdx.x) * PRE_K;
    if (i0 >= n) return;
    int m = n - i0 < PRE_K ? n - i0 : PRE_K;
    for (int w = 1; w < W; w++) {
        XYZZ<F> q[PRE_K];
        F pre[PRE_K];
        F accz = F::one();
        for (int k = 0; k < m; k++) {
            Affine<F> a = tbl[(size_t)(w - 1) * n + i0 + k];
            XYZZ<F> x = XYZZ<F>::dbl_affine(a);
            for (int d = 1; d < c; d++) x = x.dbl();
            q[k] = x;
            pre[k] = accz;
            if (!x.is_inf()) accz = accz * x.zzz;
        }
        F inv = accz.inverse();
        for (int k = m - 1; k >= 0; k--) {
            Affine<F> r;
            if (q[k].is_inf()) r = Affine<F>::inf();
            else {
                F zi = inv * pre[k];           // 1 / ZZZ_k
                inv = inv * q[k].zzz;
                F zi2 = (zi * q[k].zz).sqr();  // 1 / ZZ_k
                r.x = q[k].x * zi2; r.y = q[k].y * zi;
            }
            tbl[(size_t)w * n + i0 + k] = r;
        }
    }
}

// ---- output conversion -------------------------------------------------------------------------------
// thread per point: XYZZ -> canonical affine in Montgomery limb form (all-zero = infinity)
template <class F>
__global__ void k_to_affine(const XYZZ<F> *__restrict__ in, Affine<F> *__restrict__ out, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i].to_affine();
}

}  // namespace zkmsm
