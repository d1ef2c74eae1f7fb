// Groth16 verification on the device (SURVEY.md §8 f2): PreparedVerifyingKey, Proof::read, verify_proof for a batch,
// and Engine::pairing.  Reference boundary: core/bellman-verifier/src/verifier.rs:15-63, lib.rs:67-245 (what
// modules/zk-system calls per transaction on block import).
//
// Schedule for a batch of n proofs against one prepared key — every stage is a grid over independent work items, so a
// block's worth of transactions fills the machine even though one pairing is a long serial computation:
//   k_proof_decode_g1/g2   3n points: flags, x < q, y by square root, sign, r*P = O            (Proof::read)
//   k_jubjub_into_xy       n * n_points Jubjub encodings -> the public inputs (only for zk_groth16_verify_points_batch; jubjub.cu)
//   k_ic_partial           n * n_inputs items: x_ij * ic_j as 32 mixed additions from a per-key table of
//                          d * 2^(8w) * ic_j (d = 1..255), then k_ic_sum: ic_0 + sum_j          (the public-input MSM)
//   k_g2_prepare           n items: the 68 line coefficients of B_i                              (G2Affine::prepare)
//   k_miller               3n items: (A_i, B_i), (acc_i, -gamma), (C_i, -delta), one Miller loop each
//   k_verify_final         n items: product of the three, final exponentiation, == e(alpha, beta)
// HBM layout: per-proof arrays are structure-of-items ([item][fields]); the B_i coefficients are stored [k][i] so that
// the threads of a warp read neighbouring 288-byte records at every step of the loop; -gamma / -delta coefficients are
// one shared array (broadcast reads through L1/L2).  All of it is Fq multiply-bound (int32 pipe), not HBM-bound.
#define ZK_SEMI_HOT 1
#include <stdlib.h>
#include "internal.h"
#include "codec.cuh"
#include "pairing.cuh"

using namespace zkpair;
using zkcodec::DEC_INFINITY;
typedef Affine<Fq> G1A;
typedef Affine<Fq2> G2A;

constexpr int IC_WIN = 32, IC_DIG = 255;   // 8-bit windows of a 256-bit scalar
constexpr int PT = 64;                     // threads per block of the long-running kernels

struct zk_pvk {
    int device = 0;
    size_t n_ic = 0;
    Fq12 *alpha_beta = nullptr;
    LineCoeff *gamma = nullptr, *delta = nullptr;   // [N_COEFFS] each: prepare(-gamma_g2), prepare(-delta_g2)
    int gamma_inf = 0, delta_inf = 0;
    G1A *ic = nullptr;                              // [n_ic]
    G1A *table = nullptr;                           // [n_ic - 1][IC_WIN][IC_DIG]
    std::vector<uint8_t> image;                     // PreparedVerifyingKey::write bytes
};

// ---- small conversion kernels ----------------------------------------------------------------------------------
static __global__ void k_fq_store_be(const Fq *__restrict__ in, size_t n, uint8_t *__restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) zkcodec::fq_store_be(out + 48 * i, in[i]);
}
static __global__ void k_fq_load_be(const uint8_t *__restrict__ in, size_t n, Fq *__restrict__ out, int *__restrict__ err) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fq v;
    if (!zkcodec::fq_load_be(v, in + 48 * i, 0xff)) { atomicCAS(err, 0, (int)zkcodec::DEC_COORD); return; }
    out[i] = v;
}
// out[i * item_stride + k * coef_stride], k < N_COEFFS
static __global__ void __launch_bounds__(PT) k_g2_prepare(const G2A *__restrict__ q, size_t n, int negate, LineCoeff *__restrict__ out,
                                                          size_t item_stride, size_t coef_stride, const uint8_t *__restrict__ st, int st_stride) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (st && st[i * st_stride]) return;
    G2A p = q[i];
    if (p.is_inf()) return;
    if (negate) p.y = p.y.neg();
    g2_prepare(p, out + i * item_stride, coef_stride);
}

// ---- public-input accumulation -----------------------------------------------------------------------------------
// table[(j * IC_WIN + w) * IC_DIG + (d - 1)] = d * 2^(8 w) * ic[1 + j]
static __global__ void __launch_bounds__(PT) k_ic_table(const G1A *__restrict__ ic, size_t n_in, G1A *__restrict__ table) {
    size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= n_in * IC_WIN) return;
    size_t j = id / IC_WIN; int w = (int)(id % IC_WIN);
    XYZZ<Fq> base = XYZZ<Fq>::from_affine(ic[1 + j]);
    for (int k = 0; k < 8 * w; k++) base = base.dbl();
    G1A b = base.to_affine();
    XYZZ<Fq> acc = XYZZ<Fq>::inf();
    G1A *row = table + id * IC_DIG;
    for (int d = 0; d < IC_DIG; d++) { acc.add_mixed(b); row[d] = acc.to_affine(); }
}
static __global__ void __launch_bounds__(PT) k_ic_partial(const G1A *__restrict__ table, const uint32_t *__restrict__ inputs, size_t n, size_t n_in,
                                                          XYZZ<Fq> *__restrict__ part, int *__restrict__ err) {
    size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= n * n_in) return;
    size_t j = id % n_in;
    uint32_t k[8];
    for (int t = 0; t < 8; t++) k[t] = inputs[id * 8 + t];
    Fr kk; for (int t = 0; t < 8; t++) kk.l[t] = k[t];
    if (!Fr::canonical_lt_mod(kk)) { atomicCAS(err, 0, 1); part[id] = XYZZ<Fq>::inf(); return; }
    XYZZ<Fq> acc = XYZZ<Fq>::inf();
    const G1A *rows = table + j * IC_WIN * IC_DIG;
    for (int w = 0; w < IC_WIN; w++) {
        uint32_t d = (k[w >> 2] >> (8 * (w & 3))) & 0xff;
        if (d) acc.add_mixed(rows[(size_t)w * IC_DIG + d - 1]);
    }
    part[id] = acc;
}
static __global__ void __launch_bounds__(PT) k_ic_sum(const XYZZ<Fq> *__restrict__ part, const G1A *__restrict__ ic, size_t n, size_t n_in, G1A *__restrict__ acc_out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    XYZZ<Fq> acc = XYZZ<Fq>::from_affine(ic[0]);
    for (size_t j = 0; j < n_in; j++) acc.add(part[i * n_in + j]);
    acc_out[i] = acc.to_affine();
}

// ---- Proof::read ---------------------------------------------------------------------------------------------------
// st[3 i + slot]: 0 = ok, else a DEC_* code (DEC_INFINITY for the point at infinity); slot 0 = A, 1 = B, 2 = C
static __global__ void __launch_bounds__(PT) k_proof_decode_g1(const uint8_t *__restrict__ proofs, size_t n, G1A *__restrict__ a, G1A *__restrict__ c, uint8_t *__restrict__ st) {
    size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= 2 * n) return;
    size_t i = id >> 1; int which = (int)(id & 1);
    G1A p = G1A::inf();
    int e = zkcodec::decode_compressed(p, proofs + 192 * i + (which ? 144 : 0));
    if (!e && p.is_inf()) e = DEC_INFINITY;
    (which ? c : a)[i] = p;
    st[3 * i + (which ? 2 : 0)] = (uint8_t)e;
}
static __global__ void __launch_bounds__(PT) k_proof_decode_g2(const uint8_t *__restrict__ proofs, size_t n, G2A *__restrict__ b, uint8_t *__restrict__ st) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G2A p = G2A::inf();
    int e = zkcodec::decode_compressed(p, proofs + 192 * i + 48);
    if (!e && p.is_inf()) e = DEC_INFINITY;
    b[i] = p;
    st[3 * i + 1] = (uint8_t)e;
}

// ---- pairing kernels -----------------------------------------------------------------------------------------------
// item (type, i): type 0 = (A_i, B_i coefficients [k][i]), 1 = (acc_i, -gamma), 2 = (C_i, -delta);  f[type * n + i]
static __global__ void __launch_bounds__(PT) k_miller(size_t n, const G1A *__restrict__ a, const G1A *__restrict__ acc, const G1A *__restrict__ c,
                                                      const LineCoeff *__restrict__ coef_b, const LineCoeff *__restrict__ gamma, int gamma_inf,
                                                      const LineCoeff *__restrict__ delta, int delta_inf, const uint8_t *__restrict__ st, Fq12 *__restrict__ f) {
    size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= 3 * n) return;
    int type = (int)(id / n); size_t i = id % n;
    if (st[3 * i] | st[3 * i + 1] | st[3 * i + 2]) return;          // rejected by Proof::read: no pairing is computed
    if (type == 0) f[id] = miller_loop(a[i], coef_b + i, n, false);
    else if (type == 1) f[id] = miller_loop(acc[i], gamma, 1, gamma_inf != 0);
    else f[id] = miller_loop(c[i], delta, 1, delta_inf != 0);
}
// verdict: 1 = Ok(true), 0 = Ok(false), 2 = Proof::read -> InvalidData, 3 = Proof::read -> PointInfinity (first failing point)
static __global__ void __launch_bounds__(PT) k_verify_final(size_t n, const Fq12 *__restrict__ f, const Fq12 *__restrict__ alpha_beta,
                                                            const uint8_t *__restrict__ st, uint8_t *__restrict__ verdict) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int s = 0; s < 3; s++) {
        uint8_t e = st[3 * i + s];
        if (e) { verdict[i] = e == DEC_INFINITY ? 3 : 2; return; }
    }
    Fq12 m = mul12(mul12(f[i], f[n + i]), f[2 * n + i]), r;
    bool ok = final_exponentiation(m, r);
    verdict[i] = (ok && r == *alpha_beta) ? 1 : 0;
}
// Engine::pairing(p_i, q_i) with q_i's coefficients at coef[i * N_COEFFS ...]
static __global__ void __launch_bounds__(PT) k_pairing(size_t n, const G1A *__restrict__ p, const G2A *__restrict__ q, const LineCoeff *__restrict__ coef, Fq12 *__restrict__ out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fq12 f = miller_loop(p[i], coef + i * N_COEFFS, 1, q[i].is_inf()), r = Fq12::one();
    final_exponentiation(f, r);
    out[i] = r;
}

// ---- host side -----------------------------------------------------------------------------------------------------
static unsigned grid(size_t n, int t = PT) { return (unsigned)((n + t - 1) / t); }
static uint32_t rd_u32be(const uint8_t *p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static void wr_u32be(uint8_t *p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }
constexpr size_t COEF_BYTES = (size_t)N_COEFFS * 288;
constexpr size_t VERIFY_CHUNK = (size_t)1 << 18;      // proofs per slice of zk_groth16_verify_batch (5 GB of workspace)

extern "C" void zk_pvk_free(zk_pvk *k) {
    if (!k) return;
    cudaSetDevice(k->device);
    cudaFree(k->alpha_beta); cudaFree(k->gamma); cudaFree(k->delta); cudaFree(k->ic); cudaFree(k->table);
    delete k;
}
extern "C" size_t zk_pvk_num_inputs(const zk_pvk *k) { return k && k->n_ic ? k->n_ic - 1 : 0; }
extern "C" size_t zk_pvk_size(const zk_pvk *k) { return k ? k->image.size() : 0; }
extern "C" int zk_pvk_write(const zk_pvk *k, uint8_t *out) {
    if (!k || !out) { zk_set_error("zk_pvk_write: NULL argument"); return ZK_ERR_INVALID; }
    memcpy(out, k->image.data(), k->image.size());
    return ZK_OK;
}
static int pvk_alloc(zk_ctx *ctx, zk_pvk *k, size_t n_ic) {
    k->device = ctx->device; k->n_ic = n_ic;
    ZK_CUDA(cudaMalloc(&k->alpha_beta, sizeof(Fq12)));
    ZK_CUDA(cudaMalloc(&k->gamma, sizeof(LineCoeff) * N_COEFFS));
    ZK_CUDA(cudaMalloc(&k->delta, sizeof(LineCoeff) * N_COEFFS));
    ZK_CUDA(cudaMalloc(&k->ic, sizeof(G1A) * (n_ic ? n_ic : 1)));
    if (n_ic > 1) ZK_CUDA(cudaMalloc(&k->table, sizeof(G1A) * (n_ic - 1) * IC_WIN * IC_DIG));
    return ZK_OK;
}
static int pvk_finish(zk_ctx *ctx, zk_pvk *k) {   // the fixed-base table of ic[1..]
    if (k->n_ic > 1) {
        k_ic_table<<<grid((k->n_ic - 1) * IC_WIN), PT, 0, ctx->stream>>>(k->ic, k->n_ic - 1, k->table);
        ZK_CUDA(cudaGetLastError());
    }
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

extern "C" int zk_pvk_load(zk_ctx *ctx, const uint8_t *buf, size_t len, zk_pvk **out) {
    if (!ctx || !buf || !out) { zk_set_error("zk_pvk_load: NULL argument"); return ZK_ERR_INVALID; }
    ZK_TRY(zk_use_device(ctx));
    // layout: Fq12 | G2Prepared | G2Prepared | u32 n_ic | n_ic * G1Uncompressed
    size_t off = 576, coef_off[2] = {0, 0};
    int inf[2] = {0, 0};
    for (int g = 0; g < 2; g++) {
        if (len < off + 4) { zk_set_error("PreparedVerifyingKey: truncated"); return ZK_ERR_IO; }
        uint32_t cnt = rd_u32be(buf + off); off += 4;
        if (len < off + (size_t)cnt * 288 + 1) { zk_set_error("PreparedVerifyingKey: truncated coefficient table"); return ZK_ERR_IO; }
        coef_off[g] = off; off += (size_t)cnt * 288;
        uint8_t flag = buf[off++];
        if (flag > 1) { zk_set_error("G2Prepared: bad infinity flag %u", flag); return ZK_ERR_DECODE; }
        inf[g] = flag;
        if (!flag && cnt != (uint32_t)N_COEFFS) { zk_set_error("G2Prepared: %u coefficients, the Miller loop consumes %d", cnt, N_COEFFS); return ZK_ERR_IO; }
        if (flag) coef_off[g] = 0;
    }
    if (len < off + 4) { zk_set_error("PreparedVerifyingKey: truncated"); return ZK_ERR_IO; }
    size_t n_ic = rd_u32be(buf + off); off += 4;
    if (len < off + n_ic * 96) { zk_set_error("PreparedVerifyingKey: truncated ic"); return ZK_ERR_IO; }
    size_t total = off + n_ic * 96;
    zk_pvk *k = new zk_pvk();
    int r = pvk_alloc(ctx, k, n_ic);
    if (r) { zk_pvk_free(k); return r; }
    r = ctx->stage_a.reserve(total);
    if (r) { zk_pvk_free(k); return r; }
    uint8_t *d = ctx->stage_a.as<uint8_t>();
    int *err = ctx->d_err + 1;
    if (cudaMemcpyAsync(d, buf, total, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) { zk_pvk_free(k); zk_set_error("zk_pvk_load: copy failed"); return ZK_ERR_CUDA; }
    k_fq_load_be<<<1, 32, 0, ctx->stream>>>(d, 12, (Fq *)k->alpha_beta, err);
    for (int g = 0; g < 2; g++) {
        LineCoeff *dst = g ? k->delta : k->gamma;
        if (coef_off[g]) k_fq_load_be<<<grid(N_COEFFS * 6, 128), 128, 0, ctx->stream>>>(d + coef_off[g], (size_t)N_COEFFS * 6, (Fq *)dst, err);
        else cudaMemsetAsync(dst, 0, sizeof(LineCoeff) * N_COEFFS, ctx->stream);
    }
    if (n_ic) zkcodec::k_decode_uncompressed<Fq><<<grid(n_ic, 128), 128, 0, ctx->stream>>>(d + off, n_ic, 1, 1, k->ic, err);
    k->gamma_inf = inf[0]; k->delta_inf = inf[1];
    if (cudaGetLastError() != cudaSuccess) { zk_pvk_free(k); zk_set_error("zk_pvk_load: launch failed"); return ZK_ERR_CUDA; }
    r = zk_check_err_flag(ctx);
    if (!r) r = pvk_finish(ctx, k);
    if (r) { zk_pvk_free(k); return r; }
    k->image.assign(buf, buf + total);
    *out = k;
    return ZK_OK;
}

// one Miller loop + final exponentiation for a single pair already on the device (used for e(alpha, beta))
static int pairing_device(zk_ctx *ctx, const G1A *p, const G2A *q, size_t n, Fq12 *out) {
    ZK_TRY(ctx->v_coef.reserve(n * COEF_BYTES));
    ZK_CUDA(cudaMemsetAsync(ctx->v_coef.p, 0, n * COEF_BYTES, ctx->stream));
    k_g2_prepare<<<grid(n), PT, 0, ctx->stream>>>(q, n, 0, ctx->v_coef.as<LineCoeff>(), N_COEFFS, 1, nullptr, 0);
    k_pairing<<<grid(n), PT, 0, ctx->stream>>>(n, p, q, ctx->v_coef.as<LineCoeff>(), out);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_pvk_prepare(zk_ctx *ctx, const uint8_t *vk, size_t len, zk_pvk **out) {
    if (!ctx || !vk || !out) { zk_set_error("zk_pvk_prepare: NULL argument"); return ZK_ERR_INVALID; }
    ZK_TRY(zk_use_device(ctx));
    // VerifyingKey: alpha_g1 @0, beta_g1 @96, beta_g2 @192, gamma_g2 @384, delta_g1 @576, delta_g2 @672, u32 n_ic @864, ic @868
    if (len < 868) { zk_set_error("VerifyingKey: truncated"); return ZK_ERR_IO; }
    size_t n_ic = rd_u32be(vk + 864);
    if (len < 868 + n_ic * 96) { zk_set_error("VerifyingKey: truncated ic"); return ZK_ERR_IO; }
    size_t total = 868 + n_ic * 96;
    zk_pvk *k = new zk_pvk();
    int r = pvk_alloc(ctx, k, n_ic);
    if (!r) r = ctx->stage_a.reserve(total);
    if (!r) r = ctx->stage_b.reserve(sizeof(G1A) * 2 + sizeof(G2A) * 3);
    if (!r) r = ctx->stage_c.reserve(576 + 2 * COEF_BYTES);
    if (r) { zk_pvk_free(k); return r; }
    uint8_t *d = ctx->stage_a.as<uint8_t>();
    G1A *g1 = ctx->stage_b.as<G1A>();                       // [0] alpha, [1] delta_g1 (validated only)
    G2A *g2 = (G2A *)(g1 + 2);                              // [0] beta, [1] gamma, [2] delta
    int *err = ctx->d_err + 1;
    if (cudaMemcpyAsync(d, vk, total, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) { zk_pvk_free(k); zk_set_error("zk_pvk_prepare: copy failed"); return ZK_ERR_CUDA; }
    zkcodec::k_decode_uncompressed<Fq><<<1, 128, 0, ctx->stream>>>(d, 2, 1, 1, g1, err);                 // alpha_g1, beta_g1 (overwritten next)
    zkcodec::k_decode_uncompressed<Fq><<<1, 128, 0, ctx->stream>>>(d + 576, 1, 1, 1, g1 + 1, err);       // delta_g1
    zkcodec::k_decode_uncompressed<Fq2><<<1, 128, 0, ctx->stream>>>(d + 192, 2, 1, 1, g2, err);          // beta_g2, gamma_g2
    zkcodec::k_decode_uncompressed<Fq2><<<1, 128, 0, ctx->stream>>>(d + 672, 1, 1, 1, g2 + 2, err);      // delta_g2
    if (n_ic) zkcodec::k_decode_uncompressed<Fq><<<grid(n_ic, 128), 128, 0, ctx->stream>>>(d + 868, n_ic, 1, 1, k->ic, err);
    r = zk_check_err_flag(ctx);
    if (r) { zk_pvk_free(k); return r; }
    k_g2_prepare<<<1, PT, 0, ctx->stream>>>(g2 + 1, 1, 1, k->gamma, 0, 1, nullptr, 0);
    k_g2_prepare<<<1, PT, 0, ctx->stream>>>(g2 + 2, 1, 1, k->delta, 0, 1, nullptr, 0);
    r = pairing_device(ctx, g1, g2, 1, k->alpha_beta);
    if (r) { zk_pvk_free(k); return r; }
    // PreparedVerifyingKey::write image
    uint8_t *img = ctx->stage_c.as<uint8_t>();
    k_fq_store_be<<<1, 32, 0, ctx->stream>>>((const Fq *)k->alpha_beta, 12, img);
    k_fq_store_be<<<grid(N_COEFFS * 6, 128), 128, 0, ctx->stream>>>((const Fq *)k->gamma, (size_t)N_COEFFS * 6, img + 576);
    k_fq_store_be<<<grid(N_COEFFS * 6, 128), 128, 0, ctx->stream>>>((const Fq *)k->delta, (size_t)N_COEFFS * 6, img + 576 + COEF_BYTES);
    std::vector<uint8_t> raw(576 + 2 * COEF_BYTES);
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(raw.data(), img, raw.size(), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
        cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
        zk_pvk_free(k); zk_set_error("zk_pvk_prepare: device failure: %s", cudaGetErrorString(cudaGetLastError())); return ZK_ERR_CUDA;
    }
    k->image.resize(576 + 2 * (4 + COEF_BYTES + 1) + 4 + n_ic * 96);
    uint8_t *w = k->image.data();
    memcpy(w, raw.data(), 576); w += 576;
    for (int g = 0; g < 2; g++) {
        wr_u32be(w, N_COEFFS); w += 4;
        memcpy(w, raw.data() + 576 + g * COEF_BYTES, COEF_BYTES); w += COEF_BYTES;
        *w++ = 0;
    }
    wr_u32be(w, (uint32_t)n_ic); w += 4;
    memcpy(w, vk + 868, n_ic * 96);
    r = pvk_finish(ctx, k);
    if (r) { zk_pvk_free(k); return r; }
    *out = k;
    return ZK_OK;
}

// The verifier schedule behind zk_groth16_verify_batch_device and zk_groth16_verify_points_batch_device; all pointers are device
// pointers.  Without d_points the public inputs are d_inputs (n * n_inputs canonical Fr).  With d_points (n * n_points Jubjub
// encodings, n_inputs = 2 n_points) they are decoded first on the public-input strand into the context's workspace, and
// transactions with a rejected point get verdict 4 after the final exponentiation.
static int verify_batch(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *d_proofs, const uint64_t *d_inputs, size_t n_inputs,
                        const uint8_t *d_points, size_t n_points, uint8_t *d_verdicts) {
    const size_t chunk = VERIFY_CHUNK;
    if (n > chunk) {                   // bound the workspace (19.6 KB of B coefficients per proof): slices run back to back on the stream
        for (size_t o = 0; o < n; o += chunk) {
            size_t m = n - o < chunk ? n - o : chunk;
            ZK_TRY(verify_batch(ctx, k, m, d_proofs + 192 * o, d_points ? nullptr : d_inputs + 4 * n_inputs * o, n_inputs,
                                d_points ? d_points + 32 * n_points * o : nullptr, n_points, d_verdicts + o));
        }
        return ZK_OK;
    }
    cudaStream_t st = ctx->stream;
    uint8_t *pt_stat = nullptr;
    if (d_points) {                    // decoded inputs (64 B per point, 16-byte aligned), then one status byte per point
        ZK_TRY(ctx->v_jj.reserve(n * n_points * 65));
        d_inputs = ctx->v_jj.as<uint64_t>();
        pt_stat = ctx->v_jj.as<uint8_t>() + n * n_points * 64;
    }
    ZK_TRY(ctx->v_pts.reserve(n * (3 * sizeof(G1A) + sizeof(G2A))));
    ZK_TRY(ctx->v_stat.reserve(3 * n));
    ZK_TRY(ctx->v_coef.reserve(n * COEF_BYTES));
    ZK_TRY(ctx->v_f.reserve(3 * n * sizeof(Fq12)));
    ZK_TRY(ctx->v_part.reserve((n * n_inputs + 1) * sizeof(XYZZ<Fq>)));
    G1A *a = ctx->v_pts.as<G1A>(), *c = a + n, *acc = c + n;
    G2A *b = (G2A *)(acc + n);
    uint8_t *stt = ctx->v_stat.as<uint8_t>();
    LineCoeff *coef = ctx->v_coef.as<LineCoeff>();
    Fq12 *f = ctx->v_f.as<Fq12>();
    XYZZ<Fq> *part = ctx->v_part.as<XYZZ<Fq>>();
    // three independent strands, joined before the Miller loops: B decode + coefficients on the context's stream, A / C decode
    // and the public-input sums on the two auxiliary lanes (a small batch is latency-bound, so the strands overlap fully)
    if (!ctx->aux) { ZK_TRY(zk_ctx_create(ctx->device, nullptr, &ctx->aux)); ctx->aux->opts = ctx->opts; }
    if (!ctx->aux2) { ZK_TRY(zk_ctx_create(ctx->device, nullptr, &ctx->aux2)); ctx->aux2->opts = ctx->opts; }
    cudaStream_t s2 = ctx->aux->stream, s3 = ctx->aux2->stream;
    struct Events {                                                       // destroyed on every exit path
        cudaEvent_t e[3] = {nullptr, nullptr, nullptr};
        ~Events() { for (cudaEvent_t x : e) if (x) cudaEventDestroy(x); }     // a recorded event is released once its work completes
    } ev;
    for (cudaEvent_t &x : ev.e) ZK_CUDA(cudaEventCreateWithFlags(&x, cudaEventDisableTiming));
    ZK_CUDA(cudaEventRecord(ev.e[0], st));
    ZK_CUDA(cudaStreamWaitEvent(s2, ev.e[0], 0)); ZK_CUDA(cudaStreamWaitEvent(s3, ev.e[0], 0));
    k_proof_decode_g1<<<grid(2 * n), PT, 0, s2>>>(d_proofs, n, a, c, stt);
    ZK_CUDA(cudaEventRecord(ev.e[1], s2));
    if (d_points) zk_launch_jubjub_into_xy(s3, d_points, n * n_points, const_cast<uint64_t *>(d_inputs), pt_stat);
    if (n_inputs) k_ic_partial<<<grid(n * n_inputs), PT, 0, s3>>>(k->table, (const uint32_t *)d_inputs, n, n_inputs, part, ctx->d_err);
    k_ic_sum<<<grid(n), PT, 0, s3>>>(part, k->ic, n, n_inputs, acc);
    ZK_CUDA(cudaEventRecord(ev.e[2], s3));
    k_proof_decode_g2<<<grid(n), PT, 0, st>>>(d_proofs, n, b, stt);
    k_g2_prepare<<<grid(n), PT, 0, st>>>(b, n, 0, coef, 1, n, stt + 1, 3);
    ZK_CUDA(cudaStreamWaitEvent(st, ev.e[1], 0)); ZK_CUDA(cudaStreamWaitEvent(st, ev.e[2], 0));
    if (ctx->opts.verify_lanes) {       // six lanes per proof: one merged Miller loop, then the final exponentiation (pairing_lanes.cu)
        zk_launch_miller_lanes(st, n, a, acc, c, coef, k->gamma, k->gamma_inf, k->delta, k->delta_inf, stt, f);
        zk_launch_verify_final_lanes(st, n, f, k->alpha_beta, stt, d_verdicts);
    } else {
        k_miller<<<grid(3 * n), PT, 0, st>>>(n, a, acc, c, coef, k->gamma, k->gamma_inf, k->delta, k->delta_inf, stt, f);
        k_verify_final<<<grid(n), PT, 0, st>>>(n, f, k->alpha_beta, stt, d_verdicts);
    }
    if (d_points) zk_launch_mark_rejected_inputs(st, n, n_points, pt_stat, d_verdicts);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

static int verify_on_key_device(zk_ctx *ctx, const zk_pvk *k) {
    ZK_TRY(zk_use_device(ctx));
    if (k->device != ctx->device) { zk_set_error("prepared key lives on device %d, context on %d", k->device, ctx->device); return ZK_ERR_INVALID; }
    return ZK_OK;
}

// proofs / inputs / verdicts are device pointers
extern "C" int zk_groth16_verify_batch_device(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *d_proofs, const uint64_t *d_inputs,
                                              size_t n_inputs, uint8_t *d_verdicts) {
    if (!ctx || !k || (n && (!d_proofs || !d_verdicts)) || (n && n_inputs && !d_inputs)) { zk_set_error("zk_groth16_verify_batch: NULL argument"); return ZK_ERR_INVALID; }
    if (n_inputs + 1 != k->n_ic) {     // verifier.rs:38-40
        zk_set_error("MalformedVerifyingKey: %zu public inputs for a key with ic.len() = %zu", n_inputs, k->n_ic);
        return ZK_ERR_MALFORMED_VK;
    }
    if (!n) return ZK_OK;
    ZK_TRY(verify_on_key_device(ctx, k));
    return verify_batch(ctx, k, n, d_proofs, d_inputs, n_inputs, nullptr, 0, d_verdicts);
}

// proofs / points / verdicts are device pointers
extern "C" int zk_groth16_verify_points_batch_device(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *d_proofs, const uint8_t *d_points,
                                                     size_t n_points, uint8_t *d_verdicts) {
    if (!ctx || !k || (n && (!d_proofs || !d_verdicts)) || (n && n_points && !d_points)) { zk_set_error("zk_groth16_verify_points_batch: NULL argument"); return ZK_ERR_INVALID; }
    if (2 * n_points + 1 != k->n_ic) {
        zk_set_error("MalformedVerifyingKey: %zu public-input points (%zu inputs) for a key with ic.len() = %zu", n_points, 2 * n_points, k->n_ic);
        return ZK_ERR_MALFORMED_VK;
    }
    if (!n) return ZK_OK;
    ZK_TRY(verify_on_key_device(ctx, k));
    return verify_batch(ctx, k, n, d_proofs, nullptr, 2 * n_points, n_points ? d_points : nullptr, n_points, d_verdicts);
}

extern "C" int zk_groth16_verify_points_batch(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *proofs, const uint8_t *points, size_t n_points,
                                              uint8_t *verdicts) {
    if (!ctx || !k || (n && (!proofs || !verdicts)) || (n && n_points && !points)) { zk_set_error("zk_groth16_verify_points_batch: NULL argument"); return ZK_ERR_INVALID; }
    if (2 * n_points + 1 != k->n_ic) {
        zk_set_error("MalformedVerifyingKey: %zu public-input points (%zu inputs) for a key with ic.len() = %zu", n_points, 2 * n_points, k->n_ic);
        return ZK_ERR_MALFORMED_VK;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d_proofs, *d_pts;
    uint8_t *d_out;
    Stage io;
    io.in(proofs, d_proofs, 192 * n); io.in(points, d_pts, 32 * n * n_points); io.out(verdicts, d_out, n);
    ZK_TRY(io.up(ctx));
    ZK_TRY(zk_groth16_verify_points_batch_device(ctx, k, n, d_proofs, d_pts, n_points, d_out));
    ZK_TRY(io.down(ctx));
    return zk_check_err_flag(ctx);      // synchronises
}

extern "C" int zk_groth16_verify_batch(zk_ctx *ctx, const zk_pvk *k, size_t n, const uint8_t *proofs, const uint64_t *inputs, size_t n_inputs,
                                       uint8_t *verdicts) {
    if (!ctx || !k || (n && (!proofs || !verdicts)) || (n && n_inputs && !inputs)) { zk_set_error("zk_groth16_verify_batch: NULL argument"); return ZK_ERR_INVALID; }
    if (n_inputs + 1 != k->n_ic) {
        zk_set_error("MalformedVerifyingKey: %zu public inputs for a key with ic.len() = %zu", n_inputs, k->n_ic);
        return ZK_ERR_MALFORMED_VK;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d_proofs;
    const uint64_t *d_in;
    uint8_t *d_out;
    Stage io;
    io.in(proofs, d_proofs, 192 * n); io.in(inputs, d_in, 4 * n * n_inputs); io.out(verdicts, d_out, n);
    ZK_TRY(io.up(ctx));
    ZK_TRY(zk_groth16_verify_batch_device(ctx, k, n, d_proofs, d_in, n_inputs, d_out));
    ZK_TRY(io.down(ctx));
    return zk_check_err_flag(ctx);      // synchronises; ZK_ERR_NOT_CANONICAL if an input was >= r
}

// Engine::pairing for n (G1Uncompressed, G2Uncompressed) pairs -> n * 576 bytes (Fq12::write)
extern "C" int zk_pairing_batch(zk_ctx *ctx, size_t n, const uint8_t *g1, const uint8_t *g2, uint8_t *out) {
    if (!ctx || (n && (!g1 || !g2 || !out))) { zk_set_error("zk_pairing_batch: NULL argument"); return ZK_ERR_INVALID; }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d1, *d2;
    uint8_t *dout;
    Stage io;
    io.in(g1, d1, 96 * n); io.in(g2, d2, 192 * n); io.out(out, dout, 576 * n);
    ZK_TRY(ctx->v_pts.reserve(n * (sizeof(G1A) + sizeof(G2A))));
    ZK_TRY(ctx->v_f.reserve(n * sizeof(Fq12)));
    ZK_TRY(io.up(ctx));
    G1A *p = ctx->v_pts.as<G1A>();
    G2A *q = (G2A *)(p + n);
    int *err = ctx->d_err + 1;
    zkcodec::k_decode_uncompressed<Fq><<<grid(n, 128), 128, 0, ctx->stream>>>(d1, n, 1, 0, p, err);
    zkcodec::k_decode_uncompressed<Fq2><<<grid(n, 128), 128, 0, ctx->stream>>>(d2, n, 1, 0, q, err);
    ZK_TRY(zk_check_err_flag(ctx));
    ZK_TRY(pairing_device(ctx, p, q, n, ctx->v_f.as<Fq12>()));
    k_fq_store_be<<<grid(n * 12, 128), 128, 0, ctx->stream>>>((const Fq *)ctx->v_f.p, n * 12, dout);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}
