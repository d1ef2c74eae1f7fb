// Batched-affine bucket reduction for the Pippenger MSM (see msm.cuh for where it sits in the schedule).
//
// A mixed XYZZ addition costs 10 Montgomery products.  An AFFINE addition costs one inversion + 3 products
// (lambda = dy / dx, lambda^2, lambda * (x1 - x3)), and Montgomery's simultaneous-inversion trick shares the inversion:
// for denominators d_0 .. d_{m-1} one inverts their product once and peels the individual inverses off with 3 more
// products each — 6 products per addition.  The round-1 experiment put one binary-Euclid inversion in every THREAD
// (64 additions each): the data-dependent Euclid loops diverge inside a warp and cost more than the XYZZ addition
// they replace.  Here ONE inversion serves a whole ROUND, and a round is three kernels:
//
//   k_ba_forward   a warp owns 32 K consecutive output slots, lane l the slots w0 + 32 k + l (k < K), so the lanes of a warp
//                  touch consecutive slots at every step; classifies each pair, multiplies the denominators into a running
//                  product, parks the exclusive prefix products (k-major, coalesced); warp: two shuffle scans give every
//                  thread the product of the OTHER 31 thread totals, and the warp its total
//   k_ba_invert    ONE block over the warp totals: serial chunks + a product tree, a single field inversion (binary
//                  extended Euclid on one thread — the only serial step of the round), and the way back down
//   k_ba_backward  thread: 1 / (own total) = 1 / (warp total) x (product of the others); peels the inverse of each
//                  denominator (2 products), finishes the affine addition (3 products) and stores the sum
//
// A round halves every bucket: bucket b with m points yields ceil(m/2) points (an odd leftover is copied), so the outputs
// are again grouped by bucket and the offsets come from one scan.  A round stores its points as two planes, x[o] and y[o]:
// the next forward pass reads only the x plane, and 32 lanes on consecutive slots read and write 32 consecutive elements.
// After `levels` rounds the (short) remainders go through the XYZZ accumulation as before.  Same group elements as
// bellman's bucket sums (SURVEY.md §3.2), so the canonical result cannot change; the exceptional cases the reference's
// addition handles (P + P -> double, P + (-P) -> infinity, infinity operands; ec.rs:357-365, 394-397, 447-456, 473-476)
// are classified per pair in msm_affine_core.cuh, and the denominator of a pair that needs no division is 1, so the shared
// product is never zero.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "curve.cuh"
#include "msm_affine_core.cuh"
#include "msm_warp_scan.cuh"

namespace zkmsm {

constexpr int BA_T = 128;                     // threads per block of the forward / backward kernels
constexpr int BA_K = 32;                      // additions per thread and round
constexpr int BA_MINB = 4;                    // resident blocks per SM of the backward kernel (128 registers)
constexpr int BA_MAX_LEVELS = 8;
constexpr int BA_INV_T = 512;                 // threads of the single inversion block
constexpr uint32_t BA_NONE = 0xffffffffu;     // "no second point": the odd leftover of a bucket

// sizes_out[b] = ceil(size_in[b] / 2)
static __global__ void k_half_sizes(const uint32_t *__restrict__ off_in, uint32_t *__restrict__ sizes_out, uint32_t n_buckets) {
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n_buckets) sizes_out[b] = (off_in[b + 1] - off_in[b] + 1) >> 1;
}

template <class F>
__device__ __forceinline__ void ba_store_f(F *dst, const F &v) {
    const uint4 *s = reinterpret_cast<const uint4 *>(&v);
    uint4 *d = reinterpret_cast<uint4 *>(dst);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(F) / 16); k++) d[k] = s[k];
}
template <class F>
__device__ __forceinline__ F ba_load_f(const F *src) {
    F v;
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
    uint4 *d = reinterpret_cast<uint4 *>(&v);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(F) / 16); k++) d[k] = s[k];
    return v;
}
template <class F>
__device__ __forceinline__ F ba_ldg_f(const F *src) {
    F v;
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
    uint4 *d = reinterpret_cast<uint4 *>(&v);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(F) / 16); k++) d[k] = __ldg(s + k);
    return v;
}
// where point `code` of the round's input lives.  FIRST round: window-table row code & 0x7fffffff, stored x | y, negated when
// bit 31 is set; `in_x` is the table seen as field elements (row r: x = in_x[2r], y = in_x[2r + 1]).  Later rounds: position in
// the previous round's output planes in_x[] and in_y[].
template <class F, bool FIRST>
__device__ __forceinline__ const F *ba_x(const F *in_x, uint32_t code) { return FIRST ? in_x + 2 * (size_t)(code & 0x7fffffffu) : in_x + code; }
template <class F, bool FIRST>
__device__ __forceinline__ const F *ba_y(const F *in_x, const F *in_y, uint32_t code) { return FIRST ? ba_x<F, FIRST>(in_x, code) + 1 : in_y + code; }
template <class F, bool FIRST>
__device__ __forceinline__ Affine<F> ba_load_point(const F *in_x, const F *in_y, uint32_t code) {
    Affine<F> p;
    p.x = ba_ldg_f(ba_x<F, FIRST>(in_x, code));
    p.y = ba_ldg_f(ba_y<F, FIRST>(in_x, in_y, code));
    if (FIRST) p.y = p.y.cneg(code >> 31);
    return p;
}

// ---- which pair an output slot adds ----------------------------------------------------------------------------------
// Bucket b holds the round's outputs [off_out[b], off_out[b + 1]), made from its inputs [off_in[b], off_in[b + 1]); output j of
// the bucket adds inputs 2j and 2j + 1 (the odd leftover has no second).  A lane's slots are 32 apart: it finds the bucket of
// its first slot by binary search and walks the offsets from there (forward in the forward pass, backward in the backward
// pass), stepping over empty buckets.  In warp order the walks read neighbouring offsets, and the first round's entry codes
// of the 32 lanes are 64 consecutive words of `sorted`.
struct BaWalk {
    uint32_t b, out0, out1, in0, in1;              // bucket b: outputs [out0, out1), inputs [in0, in1)
    __device__ __forceinline__ BaWalk(const uint32_t *off_in, const uint32_t *off_out, uint32_t n_buckets, uint32_t o) {
        uint32_t lo = 0, hi = n_buckets;             // last b with off_out[b] <= o
        while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (off_out[mid] <= o) lo = mid; else hi = mid; }
        b = lo; out0 = off_out[b]; out1 = off_out[b + 1]; in0 = off_in[b]; in1 = off_in[b + 1];
    }
    __device__ __forceinline__ void forward(const uint32_t *off_in, const uint32_t *off_out, uint32_t o) {
        while (o >= out1) { b++; out0 = out1; out1 = off_out[b + 1]; in0 = in1; in1 = off_in[b + 1]; }
    }
    __device__ __forceinline__ void backward(const uint32_t *off_in, const uint32_t *off_out, uint32_t o) {
        while (o < out0) { b--; out1 = out0; out0 = off_out[b]; in1 = in0; in0 = off_in[b]; }
    }
    // the pair of slot o (in the current bucket): entry codes (FIRST round) or input positions; .y = BA_NONE for an odd leftover
    template <bool FIRST>
    __device__ __forceinline__ uint2 src(const uint32_t *sorted, uint32_t o) const {
        const uint32_t i0 = in0 + 2 * (o - out0);
        uint2 s;
        s.x = FIRST ? sorted[i0] : i0;
        s.y = i0 + 1 < in1 ? (FIRST ? sorted[i0 + 1] : i0 + 1) : BA_NONE;
        return s;
    }
};
// this lane's first slot (the warp's first slot is 32 K x the warp's index) and how many of its slots lie below `total`
__device__ __forceinline__ uint32_t ba_lane_first(size_t tid, int K) { return (uint32_t)(tid >> 5) * 32u * (uint32_t)K + (uint32_t)(tid & 31); }
__device__ __forceinline__ int ba_lane_count(uint32_t total, uint32_t oa, int K) {
    if (oa >= total) return 0;
    const uint32_t n = (total - oa + 31) >> 5;
    return n < (uint32_t)K ? (int)n : K;
}

// ---- forward ------------------------------------------------------------------------------------------------------
// in_x / in_y: see ba_x.  sorted: FIRST only (entry codes grouped by bucket).
// prefix: [(K + 1)][T_total] elements (k-major; plane K holds the thread totals).
// The denominator of an ordinary pair is x1 - x0, so this pass gathers only the x coordinates; the rare pairs that need more
// (equal x: doubling or cancellation; x = 0: possibly the point at infinity) fetch the full points.
template <class F, bool FIRST>
__global__ void __launch_bounds__(BA_T, 4) k_ba_forward(const F *__restrict__ in_x, const F *__restrict__ in_y, const uint32_t *__restrict__ sorted,
                                                         const uint32_t *__restrict__ off_in, const uint32_t *__restrict__ off_out, uint32_t n_buckets, int K,
                                                         F *__restrict__ prefix, F *__restrict__ block_totals) {
    const uint32_t total = off_out[n_buckets];
    const uint32_t n_blocks = (total + BA_T * K - 1) / (BA_T * K);
    if (blockIdx.x >= n_blocks) return;                    // the grid is sized for the host-side upper bound of `total`
    const int t = threadIdx.x;
    const size_t T_total = (size_t)gridDim.x * BA_T, tid = (size_t)blockIdx.x * BA_T + t;
    const uint32_t oa = ba_lane_first(tid, K);
    const int n = ba_lane_count(total, oa, K);
    F run = F::one();
    if (n > 0) {
        // denominators and their running product; the pair sources and their x gathers run two slots ahead
        BaWalk w(off_in, off_out, n_buckets, oa);
        uint2 s0 = w.src<FIRST>(sorted, oa), s1 = make_uint2(0, BA_NONE);
        F xa0 = ba_ldg_f(ba_x<F, FIRST>(in_x, s0.x)), xa1 = s0.y != BA_NONE ? ba_ldg_f(ba_x<F, FIRST>(in_x, s0.y)) : F::zero();
        F xb0 = F::zero(), xb1 = F::zero();
        if (n > 1) {
            w.forward(off_in, off_out, oa + 32);
            s1 = w.src<FIRST>(sorted, oa + 32);
            xb0 = ba_ldg_f(ba_x<F, FIRST>(in_x, s1.x));
            if (s1.y != BA_NONE) xb1 = ba_ldg_f(ba_x<F, FIRST>(in_x, s1.y));
        }
        for (int k = 0; k < n; k++) {
            const uint2 cur = s0;
            const F x0 = xa0, x1 = xa1;
            s0 = s1; xa0 = xb0; xa1 = xb1;
            if (k + 2 < n) {
                const uint32_t o = oa + 32u * (uint32_t)(k + 2);
                w.forward(off_in, off_out, o);
                s1 = w.src<FIRST>(sorted, o);
                xb0 = ba_ldg_f(ba_x<F, FIRST>(in_x, s1.x));
                if (s1.y != BA_NONE) xb1 = ba_ldg_f(ba_x<F, FIRST>(in_x, s1.y));
            }
            ba_store_f(prefix + (size_t)k * T_total + tid, run);
            if (cur.y == BA_NONE) continue;                 // odd leftover: copied by the backward pass
            F den = x1 - x0;
            if (den.is_zero() || x0.is_zero() || x1.is_zero()) {       // rare: decide on the full points, exactly as the backward pass will
                Affine<F> p0 = ba_load_point<F, FIRST>(in_x, in_y, cur.x), p1 = ba_load_point<F, FIRST>(in_x, in_y, cur.y);
                if (pair_classify(p0, p1, true, den) > PAIR_DBL) continue;
            }
            run = run * den;
        }
    }
    // the product of the OTHER 31 thread totals of this warp goes to plane K; the warp's total to the round's inversion
    F others, all;
    ba_warp_products(run, others, all);
    ba_store_f(prefix + (size_t)K * T_total + tid, others);
    if ((t & 31) == 0) ba_store_f(block_totals + (tid >> 5), all);
}

// ---- the round's single inversion ----------------------------------------------------------------------------------
// inv_out[i] = 1 / totals[i] for i < n = ceil(off_out[n_buckets] / (BA_T K)); scratch: n elements.
template <class F>
__global__ void __launch_bounds__(BA_INV_T) k_ba_invert(const F *__restrict__ totals, const uint32_t *__restrict__ off_out, uint32_t n_buckets, int K,
                                                        F *__restrict__ scratch, F *__restrict__ inv_out) {
    extern __shared__ unsigned char ba_smem[];
    F *node = reinterpret_cast<F *>(ba_smem);                // heap of 2 * BA_INV_T nodes
    const uint32_t total = off_out[n_buckets];
    const uint32_t n = ((total + BA_T * K - 1) / (BA_T * K)) * (BA_T / 32);       // one total per warp of the live blocks
    const int t = threadIdx.x;
    const uint32_t per = (n + BA_INV_T - 1) / BA_INV_T, c0 = t * per, c1 = c0 + per < n ? c0 + per : n;
    F run = F::one();
    for (uint32_t i = c0; i < c1; i++) { ba_store_f(scratch + i, run); run = run * ba_load_f(totals + i); }
    node[BA_INV_T + t] = run;
    for (int s = BA_INV_T / 2; s >= 1; s >>= 1) {
        __syncthreads();
        if (t < s) node[s + t] = node[2 * (s + t)] * node[2 * (s + t) + 1];
    }
    __syncthreads();
    if (t == 0) node[1] = node[1].inverse();                  // every factor is non-zero by construction (pair_classify)
    for (int s = 1; s < BA_INV_T; s <<= 1) {
        __syncthreads();
        if (t < s) {
            F inv = node[s + t], l = node[2 * (s + t)], r = node[2 * (s + t) + 1];
            node[2 * (s + t)] = inv * r;
            node[2 * (s + t) + 1] = inv * l;
        }
    }
    __syncthreads();
    F inv = node[BA_INV_T + t];
    for (uint32_t i = c1; i-- > c0;) {
        F v = ba_load_f(totals + i);
        ba_store_f(inv_out + i, inv * ba_load_f(scratch + i));
        inv = inv * v;
    }
}

// ---- backward ------------------------------------------------------------------------------------------------------
// Walks the lane's slots from the last to the first and stores each sum as out_x[o], out_y[o].
template <class F, bool FIRST, int MINB>
__global__ void __launch_bounds__(BA_T, MINB) k_ba_backward(const F *__restrict__ in_x, const F *__restrict__ in_y, const uint32_t *__restrict__ sorted,
                                                             const uint32_t *__restrict__ off_in, const uint32_t *__restrict__ off_out, uint32_t n_buckets, int K,
                                                             const F *__restrict__ prefix, const F *__restrict__ block_inv,
                                                             F *__restrict__ out_x, F *__restrict__ out_y) {
    constexpr int PV = (int)(sizeof(Affine<F>) / 16), FV = (int)(sizeof(F) / 16);     // a slot = two points + one prefix element
    extern __shared__ unsigned char ba_smem[];
    uint4 *stage = reinterpret_cast<uint4 *>(ba_smem);
    const uint32_t total = off_out[n_buckets];
    const uint32_t n_blocks = (total + BA_T * K - 1) / (BA_T * K);
    if (blockIdx.x >= n_blocks) return;
    const int t = threadIdx.x;
    const size_t T_total = (size_t)gridDim.x * BA_T, tid = (size_t)blockIdx.x * BA_T + t;
    const uint32_t oa = ba_lane_first(tid, K);
    const int n = ba_lane_count(total, oa, K);
    if (n == 0) return;
    // inverse of this thread's total = (inverse of the warp's total) x (product of the other 31 totals of the warp)
    F inv = ba_load_f(block_inv + (tid >> 5)) * ba_load_f(prefix + (size_t)K * T_total + tid);
    // software pipeline: while addition k is finished, the operands of k - 1 (two points, one prefix product) stream into
    // this thread's shared-memory slot with cp.async — the gather latency hides behind five Montgomery products
    uint4 *slot = stage + t;                                  // vector v of the slot lives at stage[v * BA_T + t]: conflict-free
    auto copy = [&](int v, const F *src) {
        const uint4 *s = reinterpret_cast<const uint4 *>(src);
#pragma unroll
        for (int u = 0; u < FV; u++)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(slot + (v + u) * BA_T)), "l"(s + u) : "memory");
    };
    auto prefetch = [&](int k, uint2 src) {
        const uint32_t c1 = src.y == BA_NONE ? src.x : src.y;
        copy(0, ba_x<F, FIRST>(in_x, src.x));
        copy(FV, ba_y<F, FIRST>(in_x, in_y, src.x));
        copy(PV, ba_x<F, FIRST>(in_x, c1));
        copy(PV + FV, ba_y<F, FIRST>(in_x, in_y, c1));
        copy(2 * PV, prefix + (size_t)k * T_total + tid);
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    BaWalk w(off_in, off_out, n_buckets, oa + 32u * (uint32_t)(n - 1));
    uint2 src = w.src<FIRST>(sorted, oa + 32u * (uint32_t)(n - 1));
    prefetch(n - 1, src);
    for (int k = n; k-- > 0;) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        Affine<F> p0, p1;
        F pre;
        {
            uint4 *d0 = reinterpret_cast<uint4 *>(&p0), *d1 = reinterpret_cast<uint4 *>(&p1), *d2 = reinterpret_cast<uint4 *>(&pre);
#pragma unroll
            for (int v = 0; v < PV; v++) { d0[v] = slot[v * BA_T]; d1[v] = slot[(PV + v) * BA_T]; }
#pragma unroll
            for (int v = 0; v < FV; v++) d2[v] = slot[(2 * PV + v) * BA_T];
        }
        const uint2 cur = src;
        if (k > 0) {
            const uint32_t o = oa + 32u * (uint32_t)(k - 1);
            w.backward(off_in, off_out, o);
            src = w.src<FIRST>(sorted, o);
            prefetch(k - 1, src);
        }
        const bool has1 = cur.y != BA_NONE;
        if (FIRST) { p0.y = p0.y.cneg(cur.x >> 31); if (has1) p1.y = p1.y.cneg(cur.y >> 31); }
        if (!has1) p1 = Affine<F>::inf();
        F den;
        const int mode = pair_classify(p0, p1, has1, den);
        F dinv = F::one();
        if (mode <= PAIR_DBL) { dinv = inv * pre; inv = inv * den; }
        Affine<F> r = pair_finish(mode, p0, p1, dinv);
        const uint32_t o = oa + 32u * (uint32_t)k;
        ba_store_f(out_x + o, r.x);
        ba_store_f(out_y + o, r.y);
    }
}

// dynamic shared memory of the three kernels
template <class F> constexpr size_t ba_smem_forward() { return 0; }
template <class F> constexpr size_t ba_smem_backward() { return (size_t)BA_T * (2 * sizeof(Affine<F>) + sizeof(F)); }
template <class F> constexpr size_t ba_smem_invert() { return 2 * BA_INV_T * sizeof(F); }

}  // namespace zkmsm
