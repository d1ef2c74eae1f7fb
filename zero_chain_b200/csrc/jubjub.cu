// Jubjub public-input decoding on the device (jubjub.cuh): zk_jubjub_into_xy, and the two launches the point-taking verifier
// (pairing.cu, zk_groth16_verify_points_batch) adds around its pairing check.  One thread per 32-byte encoding: the work is
// ~4 k Fr products per point (Tonelli-Shanks ~0.9 k, [r_J] P ~3.1 k), all of it in registers.
//
// The translation unit holds only Fr arithmetic, so it is compiled with everything inlined (ZK_HOT): the cold-path
// convention of a real call boundary around each product would put the point and the square-root state on a stack frame.
#define ZK_HOT 1
#include "internal.h"
#include "jubjub.cuh"

constexpr int JT = 128;   // threads per block

// xy[2 p], xy[2 p + 1]: canonical x, y of point p (4 LE u64 each, the layout k_ic_partial reads); st[p]: zkjj::Status
static __global__ void __launch_bounds__(JT) k_jubjub_into_xy(const uint8_t *__restrict__ enc, size_t n, uint32_t *__restrict__ xy,
                                                              uint8_t *__restrict__ st) {
    size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    uint32_t w[8];
    const uint8_t *b = enc + 32 * p;       // byte loads: a device pointer passed in by the caller need not be word aligned
#pragma unroll
    for (int i = 0; i < 8; i++)
        w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
    Fr x, y;
    int s = zkjj::jubjub_into_xy(w, x, y);
    uint4 *o = reinterpret_cast<uint4 *>(xy + 16 * p);
    o[0] = make_uint4(x.l[0], x.l[1], x.l[2], x.l[3]);
    o[1] = make_uint4(x.l[4], x.l[5], x.l[6], x.l[7]);
    o[2] = make_uint4(y.l[0], y.l[1], y.l[2], y.l[3]);
    o[3] = make_uint4(y.l[4], y.l[5], y.l[6], y.l[7]);
    st[p] = (uint8_t)s;
}

// verdict 4 for every transaction with a rejected point: the reference builds the public inputs before Proof::read
// (modules/zk-system/src/lib.rs:69-103), so this overrides 2 / 3 as well as the pairing outcome
static __global__ void k_mark_rejected_inputs(size_t n, size_t n_points, const uint8_t *__restrict__ st, uint8_t *__restrict__ verdict) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t bad = 0;
    for (size_t j = 0; j < n_points; j++) bad |= st[i * n_points + j];
    if (bad) verdict[i] = ZK_VERDICT_INPUT_REJECTED;
}

void zk_launch_jubjub_into_xy(cudaStream_t s, const uint8_t *d_enc, size_t n, uint64_t *d_xy, uint8_t *d_status) {
    if (n) k_jubjub_into_xy<<<(unsigned)((n + JT - 1) / JT), JT, 0, s>>>(d_enc, n, reinterpret_cast<uint32_t *>(d_xy), d_status);
}
void zk_launch_mark_rejected_inputs(cudaStream_t s, size_t n, size_t n_points, const uint8_t *d_status, uint8_t *d_verdicts) {
    if (n) k_mark_rejected_inputs<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(n, n_points, d_status, d_verdicts);
}

extern "C" int zk_jubjub_into_xy(zk_ctx *ctx, size_t n, const uint8_t *points, uint64_t *xy, uint8_t *status) {
    if (!ctx || (n && (!points || !xy || !status))) { zk_set_error("zk_jubjub_into_xy: NULL argument"); return ZK_ERR_INVALID; }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d_in;
    uint64_t *d_xy;
    uint8_t *d_st;
    Stage io;
    io.in(points, d_in, 32 * n); io.out(xy, d_xy, 8 * n); io.out(status, d_st, n);
    ZK_TRY(io.up(ctx));
    zk_launch_jubjub_into_xy(ctx->stream, d_in, n, d_xy, d_st);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}
