// RedJubjub signature verification on the device (redjubjub.cuh): zk_redjubjub_verify_batch and its _device form.  One
// thread per signature: BLAKE2b over rbar || msg, two Point::reads and one shared doubling chain, ~6 k Fr products, all of
// it in registers.
//
// Like jubjub.cu, the translation unit holds only Fr / Fs arithmetic and is compiled with everything inlined (ZK_HOT).
#define ZK_HOT 1
#include "internal.h"
#include "redjubjub.cuh"

constexpr int RT = 128;             // threads per block
constexpr int RJ_BLOCKS_PER_SM = 8; // grid cap: larger batches loop over the grid

static __device__ __forceinline__ void load_le_words(const uint8_t *b, uint32_t *w, int n) {
#pragma unroll
    for (int i = 0; i < n; i++)     // byte loads: a device pointer passed in by the caller need not be word aligned
        w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
}

// message i = msgs[off[i] - base .. off[i + 1] - base)
static __global__ void __launch_bounds__(RT) k_redjubjub_verify(size_t n, const uint8_t *__restrict__ vks, const uint8_t *__restrict__ sigs,
                                                                const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off,
                                                                uint64_t base, uint8_t *__restrict__ verdicts) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t vk[8], sig[16];
        load_le_words(vks + 32 * i, vk, 8);
        load_le_words(sigs + 64 * i, sig, 16);
        const uint64_t o0 = off[i] - base, o1 = off[i + 1] - base;
        verdicts[i] = (uint8_t)zkrj::redjubjub_verify(vk, sig, msgs + o0, o1 - o0);
    }
}

static void launch_verify(zk_ctx *ctx, size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *off,
                          uint64_t base, uint8_t *verdicts) {
    const size_t cap = (size_t)(ctx->sm_count > 0 ? ctx->sm_count : 1) * RJ_BLOCKS_PER_SM;
    const size_t blocks = (n + RT - 1) / RT < cap ? (n + RT - 1) / RT : cap;
    k_redjubjub_verify<<<(unsigned)blocks, RT, 0, ctx->stream>>>(n, vks, sigs, msgs, off, base, verdicts);
}

extern "C" int zk_redjubjub_verify_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_vks, const uint8_t *d_sigs, const uint8_t *d_msgs,
                                                const uint64_t *d_msg_off, uint8_t *d_verdicts) {
    if (!ctx || (n && (!d_vks || !d_sigs || !d_msgs || !d_msg_off || !d_verdicts))) {
        zk_set_error("zk_redjubjub_verify_batch_device: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    launch_verify(ctx, n, d_vks, d_sigs, d_msgs, d_msg_off, 0, d_verdicts);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_redjubjub_verify_batch(zk_ctx *ctx, size_t n, const uint8_t *vks, const uint8_t *sigs, const uint8_t *msgs,
                                         const uint64_t *msg_off, uint8_t *verdicts) {
    if (!ctx || (n && (!vks || !sigs || !msgs || !msg_off || !verdicts))) {
        zk_set_error("zk_redjubjub_verify_batch: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    for (size_t i = 0; i < n; i++)
        if (msg_off[i + 1] < msg_off[i]) {   // msgs ends at msg_off[n]: a decreasing offset puts a message past its end
            zk_set_error("zk_redjubjub_verify_batch: msg_off[%zu] = %llu > msg_off[%zu] = %llu", i, (unsigned long long)msg_off[i], i + 1,
                         (unsigned long long)msg_off[i + 1]);
            return ZK_ERR_INVALID;
        }
    ZK_TRY(zk_use_device(ctx));
    const uint64_t base = msg_off[0];       // the messages go up from msgs[base]; the kernel subtracts base from each offset
    const uint8_t *d_vks, *d_sigs, *d_msgs;
    const uint64_t *d_off;
    uint8_t *d_ver;
    Stage io;
    io.in(msg_off, d_off, n + 1); io.in(vks, d_vks, 32 * n); io.in(sigs, d_sigs, 64 * n); io.in(msgs + base, d_msgs, msg_off[n] - base);
    io.out(verdicts, d_ver, n);
    ZK_TRY(io.up(ctx));
    launch_verify(ctx, n, d_vks, d_sigs, d_msgs, d_off, base, d_ver);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}
