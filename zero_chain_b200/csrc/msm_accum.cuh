// Bucket accumulation kernel of the Pippenger MSM (see msm.cuh for the whole schedule).
// Kept in its own header so the hot translation unit (msm_hot.cu, compiled with ZK_HOT: Montgomery
// products and the mixed addition fully inlined) and the cold one (G2) share one source.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "curve.cuh"

namespace zkmsm {

constexpr int TASK_LEN_MAX = 64;          // target upper bound of mixed additions per accumulate task
constexpr int TASK_LEN_MIN = 16;         // shorter tasks make the per-bucket combine (serial point additions) the bottleneck of small MSMs

template <class F>
__device__ __forceinline__ Affine<F> load_affine(const Affine<F> *__restrict__ p) {
    Affine<F> r;
    const uint4 *s = reinterpret_cast<const uint4 *>(p);
    uint4 *d = reinterpret_cast<uint4 *>(&r);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(Affine<F>) / 16); k++) d[k] = __ldg(s + k);
    return r;
}
// MINB = minimum resident blocks per SM (register budget: 2 -> <=255 regs, 3 -> 168, 4 -> 128)
// Points: ys == nullptr -> xs holds affine rows x | y (row r: x = xs[2r], y = xs[2r + 1]: bases or window tables); otherwise
// two planes x = xs[i], y = ys[i] (the last batched-affine round's outputs, msm_batchaff.cuh).
template <class F, int MINB>
__global__ void __launch_bounds__(128, MINB) k_accumulate(const F *__restrict__ xs, const F *__restrict__ ys, const uint32_t *__restrict__ sorted,
                                                    const uint32_t *__restrict__ bucket_off, const uint32_t *__restrict__ task_off,
                                                    uint32_t n_buckets, const uint32_t *__restrict__ order, XYZZ<F> *__restrict__ partials) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n_tasks = task_off[n_buckets];
    if (t >= n_tasks) return;
    if (order) t = order[t];          // tasks issued by decreasing length (k_len_place): equal work inside a warp
    // bucket of task t: last b with task_off[b] <= t
    uint32_t lo = 0, hi = n_buckets;
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (task_off[mid] <= t) lo = mid; else hi = mid; }
    uint32_t b = lo, s = t - task_off[b];
    // split the bucket EVENLY over its tasks (all tasks of a bucket within one entry of each other), so the
    // lanes of a warp run the same number of additions instead of full tasks next to a short remainder
    uint32_t nt = task_off[b + 1] - task_off[b], b0 = bucket_off[b], size = bucket_off[b + 1] - b0;
    uint32_t len = (size + nt - 1) / nt;
    uint32_t e0 = b0 + s * len, e1 = e0 + len;
    if (e1 > b0 + size) e1 = b0 + size;
    if (e0 >= e1) { partials[t] = XYZZ<F>::inf(); return; }
    XYZZ<F> acc = XYZZ<F>::inf();
    // The next point is prefetched with cp.async into a per-thread shared-memory slot while the current mixed
    // addition runs: the gather latency is hidden without holding a second point (24+ registers) live.
    // sorted == nullptr: the inputs are already-reduced affine points indexed by position (no sign)
    constexpr int VEC = (int)(sizeof(Affine<F>) / 16), FV = (int)(sizeof(F) / 16);
    __shared__ uint4 stage[128 * VEC];
    uint4 *slot = stage + threadIdx.x * VEC;
    const uint32_t slot_addr = (uint32_t)__cvta_generic_to_shared(slot);
    auto prefetch = [&](uint32_t c) {
        const F *px = ys ? xs + c : xs + 2 * (size_t)(c & 0x7fffffffu), *py = ys ? ys + c : px + 1;
        const uint4 *sx = reinterpret_cast<const uint4 *>(px), *sy = reinterpret_cast<const uint4 *>(py);
#pragma unroll
        for (int k = 0; k < FV; k++) {
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slot_addr + 16u * k), "l"(sx + k) : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slot_addr + 16u * (FV + k)), "l"(sy + k) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    uint32_t code = sorted ? sorted[e0] : e0;
    prefetch(code);
    for (uint32_t e = e0; e < e1; e++) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        Affine<F> p;
        {
            uint4 *d = reinterpret_cast<uint4 *>(&p);
#pragma unroll
            for (int k = 0; k < VEC; k++) d[k] = slot[k];
        }
        bool neg = code >> 31;
        if (e + 1 < e1) { code = sorted ? sorted[e + 1] : e + 1; prefetch(code); }
        p.y = p.y.cneg(neg);
        acc.add_mixed(p);
    }
    partials[t] = acc;
}
}  // namespace zkmsm
