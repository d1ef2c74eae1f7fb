// Radix-2 NTT over the BLS12-381 scalar field Fr for sm_90a (H100).
//
// Replaces upstream bellman 0.1.0 `EvaluationDomain::{fft, ifft, coset_fft, icoset_fft}` (SURVEY.md
// §3.2, §8 a7; reached from create_proof, reference call site core/proofs/src/confidential.rs:149).
// Same definition — out[k] = sum_j a[j] w^(jk), w = ROOT_OF_UNITY^(2^(32-log_n)) (fr.rs:47-55),
// coset generator 7 (fr.rs:38-44), ifft scaled by m^-1 — so results are bit-identical; the schedule
// is GPU-first instead of bellman's serial bit-reversal + log n global butterfly rounds:
//
//   four-step split N = N1 x N2 (log N1 = floor(k/2)): two kernels, each doing a complete
//   sub-transform of <= 2048 points in SHARED MEMORY (decimation in frequency, in place),
//     pass A  columns (stride N2): [x g^i] -> N1-point DFT -> x w^(n2 m1) -> back in place
//     pass B  rows (contiguous):   N2-point DFT -> [x g^-i m^-1 | x m^-1] -> transposed store
//   The bit-reversal is never materialised: each pass reads its DIF result out of shared memory in
//   bit-reversed order, and adjacent columns / rows are grouped per block so global accesses are
//   COLS*32 B / ROWS*32 B contiguous.  Twiddles come from per-size tables (w^i, g^i, g^-i/m) built
//   once per context and log_n; the kernel is bound by the Fr Montgomery products
//   (k/2 + ~1.1 per element), not by HBM (3 x 32 B per element per pass).
//   A batch of transforms of the same size (the prover's 7 per proof) is one launch (grid.y).
#define ZK_HOT 1
#include "internal.h"
#include "field.cuh"
#include "tma.cuh"

namespace {

constexpr int NTT_THREADS = 256;
constexpr int MAX_TILE_LOG = 11;    // 2048 elements * 32 B = 64 KB of shared memory

// Fr constants in Montgomery form (fr.rs:38-55)
__device__ __forceinline__ Fr fr_generator() {
    Fr g; const uint32_t v[8] = {0xfffffff1u, 0x0000000eu, 0x00189c0fu, 0x17e363d3u, 0x6f8457b0u, 0xff9c5787u, 0x8fc5a8c4u, 0x35133220u};
    for (int i = 0; i < 8; i++) g.l[i] = v[i];
    return g;
}
__device__ __forceinline__ Fr fr_root_of_unity() {
    Fr g; const uint32_t v[8] = {0x5f0e466au, 0xb9b58d8cu, 0x1819d7ecu, 0x5b1b4c80u, 0x52a31e64u, 0x0af53ae3u, 0x19e9b27bu, 0x5bf3addau};
    for (int i = 0; i < 8; i++) g.l[i] = v[i];
    return g;
}
__device__ __forceinline__ Fr fr_generator_inv() {   // 7^-1
    Fr g; const uint32_t v[8] = {0xdb6db6dcu, 0xdb6db6dau, 0xdb6cc6dau, 0xe6b5824au, 0x05810db9u, 0xf8b356e0u, 0x60ec4796u, 0x66d0f1e6u};
    for (int i = 0; i < 8; i++) g.l[i] = v[i];
    return g;
}
__device__ __forceinline__ Fr fr_inv2() {            // 2^-1
    Fr g; const uint32_t v[8] = {0xffffffffu, 0x00000000u, 0x0001a401u, 0xac425bfdu, 0xf65e27fau, 0xccc627f7u, 0xd66282b7u, 0x0c1258acu};
    for (int i = 0; i < 8; i++) g.l[i] = v[i];
    return g;
}
__device__ __forceinline__ Fr fr_pow_u64(Fr base, uint64_t e) {
    Fr acc = Fr::one();
    while (e) { if (e & 1) acc = acc * base; base = base * base; e >>= 1; }
    return acc;
}
__device__ __forceinline__ Fr load_fr(const Fr *p) {
    const uint4 *s = reinterpret_cast<const uint4 *>(p);
    uint4 a = s[0], b = s[1];
    Fr r; r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}
__device__ __forceinline__ void store_fr(Fr *p, const Fr &v) {
    uint4 *d = reinterpret_cast<uint4 *>(p);
    d[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    d[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}

// tables: W[i] = w^i, G[i] = g^i, GI[i] = g^-i * m^-1, i < N;  consts[0] = m^-1, consts[1] = (g^m - 1)^-1
__global__ void k_ntt_tables(Fr *W, Fr *G, Fr *GI, Fr *consts, unsigned log_n) {
    size_t n = (size_t)1 << log_n;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr w = fr_root_of_unity();
    for (unsigned k = log_n; k < 32; k++) w = w * w;
    Fr g = fr_generator();
    Fr minv = fr_pow_u64(fr_inv2(), log_n);      // (2^log_n)^-1
    store_fr(W + i, fr_pow_u64(w, i));
    store_fr(G + i, fr_pow_u64(g, i));
    store_fr(GI + i, fr_pow_u64(fr_generator_inv(), i) * minv);
    if (i == 0) {
        store_fr(consts, minv);
        store_fr(consts + 1, (fr_pow_u64(g, n) - Fr::one()).inverse());   // divide_by_z_on_coset: (g^m - 1)^-1
    }
}

__device__ __forceinline__ unsigned bitrev(unsigned x, int bits) { return bits ? (__brev(x) >> (32 - bits)) : 0; }

// Geometry of one pass.  A "sub-array" is a contiguous run of 2^log_sub elements transformed on its own
// (the whole vector for sizes <= 2^22; one row of 2^22 for larger sizes, whose root is w_N^(2^tw_shift)).
struct PassGeom {
    unsigned log_n;      // size of the whole transform (table index space)
    unsigned log_sub;    // size of the sub-array this pass works in
    int l1;              // columns pass: log of the column length; rows pass: log of the number of rows in the sub-array
    int tw_shift;        // log_n - log_sub: sub-array twiddles are table entries scaled by 2^tw_shift
    int y_is_row;        // blockIdx.y selects a row of the outer split (1) or a batch item (0)
    int out_shift;       // rows pass with y_is_row: global out index = blockIdx.y + (o_sub << out_shift)
};

// In-place decimation-in-frequency transform of `cnt` independent tiles of 2^lb points held in
// shared memory (tile t at sm + t * 2^lb).  Twiddle for the butterfly (i, i+h) of a 2h-group is
// w_sub^(j * sub/(2h)), j = i mod h; inverse transforms index the table from the other end.
__device__ __forceinline__ void smem_dif(Fr *sm, int lb, int cnt, const Fr *__restrict__ W, const PassGeom &g, bool inverse) {
    const unsigned n_mask = g.log_n >= 32 ? 0xffffffffu : ((1u << g.log_n) - 1);
    const int half_total = (cnt << lb) >> 1;
    for (int s = lb - 1; s >= 0; s--) {
        const int h = 1 << s;
        __syncthreads();
        for (int q = threadIdx.x; q < half_total; q += NTT_THREADS) {
            int j = q & (h - 1);
            int i = ((q >> s) << (s + 1)) | j;          // covers all tiles: tile size is a multiple of 2h
            Fr a = sm[i], b = sm[i + h];
            unsigned e = (unsigned)j << (g.log_n - s - 1);      // j * N / 2h  (independent of the sub-array size)
            if (inverse) e = (0u - e) & n_mask;
            Fr d = a - b;
            sm[i] = a + b;
            sm[i + h] = s == 0 ? d : d * load_fr(W + e);   // j == 0 when h == 1: twiddle 1
        }
    }
    __syncthreads();
}

// columns pass over each sub-array viewed as [2^l1][2^(log_sub-l1)]; block handles 2^cols_log adjacent columns.
__global__ void __launch_bounds__(NTT_THREADS) k_ntt_cols(const Fr *__restrict__ in, Fr *__restrict__ out, PassGeom g, int cols_log,
                                                          const Fr *__restrict__ W, const Fr *__restrict__ G, int coset_in, int inverse) {
    extern __shared__ __align__(128) unsigned char smraw[];
    Fr *sm = reinterpret_cast<Fr *>(smraw);
    const int l1 = g.l1, l2 = g.log_sub - l1, N1 = 1 << l1, cols = 1 << cols_log;
    const size_t N2 = (size_t)1 << l2;
    const size_t base = (size_t)blockIdx.y << g.log_sub;
    const Fr *x = in + base;
    Fr *y = out + base;
    const size_t c0 = (size_t)blockIdx.x << cols_log;
    const int total = N1 << cols_log;
    const unsigned n_mask = g.log_n >= 32 ? 0xffffffffu : ((1u << g.log_n) - 1);
    // load: consecutive threads take consecutive columns of one row (cols*32 B contiguous); tile layout [col][n1]
    for (int q = threadIdx.x; q < total; q += NTT_THREADS) {
        int col = q & (cols - 1), n1 = q >> cols_log;
        size_t idx = (size_t)n1 * N2 + c0 + col;
        Fr v = load_fr(x + idx);
        if (coset_in) v = v * load_fr(G + idx);             // coset scaling only where the sub-array is the whole transform
        sm[(col << l1) + n1] = v;
    }
    smem_dif(sm, l1, cols, W, g, inverse != 0);
    // store: frequency m1 sits at position bitrev(m1); multiply by the four-step twiddle w_sub^(n2*m1)
    for (int q = threadIdx.x; q < total; q += NTT_THREADS) {
        int col = q & (cols - 1), m1 = q >> cols_log;
        size_t n2 = c0 + col;
        Fr v = sm[(col << l1) + bitrev(m1, l1)];
        unsigned e = (unsigned)(((n2 * (size_t)m1) << g.tw_shift) & n_mask);
        if (inverse) e = (0u - e) & n_mask;
        if (e) v = v * load_fr(W + e);
        store_fr(y + (size_t)m1 * N2 + n2, v);
    }
}

// rows pass: each sub-array viewed as [2^l1][2^(log_sub-l1)]; block handles 2^rows_log adjacent rows; frequency
// (m1, m2) goes to sub-array index m1 + 2^l1 * m2, i.e. the transposed position that makes the output natural order.
// post: 0 none, 1 multiply by consts[0] (m^-1), 2 multiply by GI[global out index] (g^-i m^-1)
__global__ void __launch_bounds__(NTT_THREADS) k_ntt_rows(const Fr *__restrict__ in, Fr *__restrict__ out, PassGeom g, int rows_log,
                                                          const Fr *__restrict__ W, const Fr *__restrict__ G, const Fr *__restrict__ GI,
                                                          const Fr *__restrict__ consts, int coset_in, int inverse, int post) {
    extern __shared__ __align__(128) unsigned char smraw[];
    Fr *sm = reinterpret_cast<Fr *>(smraw);
    const int l1 = g.l1, l2 = g.log_sub - l1, N2 = 1 << l2, rows = 1 << rows_log;
    const size_t N1 = (size_t)1 << l1;
    const size_t base = (size_t)blockIdx.y << g.log_sub;
    const Fr *x = in + base;
    const size_t r0 = (size_t)blockIdx.x << rows_log;
    const int total = N2 << rows_log;
    if (!coset_in) {
        // the block's rows are one contiguous run of total*32 B: stage it with bulk asynchronous copies
        // (TMA engine, mbarrier completion) instead of per-thread loads
        __shared__ uint64_t bar;
        const uint32_t bytes = (uint32_t)total * 32u, CH = 16384u;
        if (threadIdx.x == 0) zktma::mbar_init(&bar, 1);
        __syncthreads();
        if (threadIdx.x == 0) {
            zktma::mbar_expect_tx(&bar, bytes);
            const unsigned char *src = reinterpret_cast<const unsigned char *>(x + (r0 << l2));
            for (uint32_t o = 0; o < bytes; o += CH) zktma::bulk_load(smraw + o, src + o, bytes - o < CH ? bytes - o : CH, &bar);
        }
        zktma::mbar_wait(&bar, 0);
    } else {
        for (int q = threadIdx.x; q < total; q += NTT_THREADS) {     // coset scaling on load (only when there is no columns pass)
            size_t idx = (r0 << l2) + q;
            sm[q] = load_fr(x + idx) * load_fr(G + idx);
        }
    }
    smem_dif(sm, l2, rows, W, g, inverse != 0);
    Fr scale = Fr::one();
    if (post == 1) scale = load_fr(consts);
    for (int q = threadIdx.x; q < total; q += NTT_THREADS) {     // consecutive threads: consecutive m1 of one m2
        int row = q & (rows - 1), m2 = q >> rows_log;
        Fr v = sm[(row << l2) + bitrev(m2, l2)];
        size_t o_sub = (r0 + row) + N1 * (size_t)m2;
        size_t o = g.y_is_row ? (size_t)blockIdx.y + (o_sub << g.out_shift) : base + o_sub;
        if (post == 1) v = v * scale;
        else if (post == 2) v = v * load_fr(GI + (g.y_is_row ? o : o_sub));   // table index = position inside the transform
        store_fr(out + o, v);
    }
}

}  // namespace

// Twiddle tables (w^i, g^i, g^-i / m) live in the CONTEXT that uses them (internal.h: zk_ctx::ntt_slots): a context is single-threaded
// and owns one stream, so building a table, rebuilding a slot for another size and reading it are all ordered on that stream —
// no cross-stream or cross-thread hazards, nothing process-global, and zk_ctx_destroy frees them.  Least-recently-used slot is recycled.
static int get_tables(zk_ctx *ctx, unsigned log_n, NttSlot **out) {
    NttSlot *victim = nullptr;
    ctx->ntt_clock++;
    for (NttSlot &sl : ctx->ntt_slots)
        if (sl.valid && sl.log_n == log_n) { sl.last_use = ctx->ntt_clock; *out = &sl; return ZK_OK; }
    for (NttSlot &sl : ctx->ntt_slots) {            // an empty slot if there is one, else the least recently used
        if (!sl.valid) { victim = &sl; break; }
        if (!victim || sl.last_use < victim->last_use) victim = &sl;
    }
    size_t n = (size_t)1 << log_n;
    victim->valid = false;
    ZK_TRY(victim->w.reserve(n * 32)); ZK_TRY(victim->g.reserve(n * 32)); ZK_TRY(victim->gi.reserve(n * 32)); ZK_TRY(victim->consts.reserve(64));
    k_ntt_tables<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(victim->w.as<Fr>(), victim->g.as<Fr>(), victim->gi.as<Fr>(),
                                                                       victim->consts.as<Fr>(), log_n);
    ZK_CUDA(cudaGetLastError());
    victim->log_n = log_n; victim->valid = true; victim->last_use = ctx->ntt_clock;
    *out = victim;
    return ZK_OK;
}

// `batch` transforms of 2^log_n contiguous elements each, in place in d_data.
//   log_n <= 11          one rows pass, the whole vector in one shared-memory tile (in place)
//   12 <= log_n <= 22    columns pass data -> tmp, rows pass tmp -> data
//   log_n > 22           outer split N = 2^(log_n-22) x 2^22: columns pass over the outer dimension, then every 2^22 row
//                        gets the two passes above with the root w^(2^(log_n-22)) and a transposed final store; a batch runs
//                        these three passes once per vector (grid.y already indexes the rows), all through the one ntt_tmp
int zk_ntt_run(zk_ctx *ctx, void *d_data, unsigned log_n, int mode, size_t batch) {
    if (log_n > 32) { zk_set_error("PolynomialDegreeTooLarge: log_n = %u", log_n); return ZK_ERR_POLY_DEGREE_TOO_LARGE; }
    if (log_n > 28) { zk_set_error("NTT sizes above 2^28 are not supported by this build (twiddle tables would need %llu GB)", (unsigned long long)(96ull << (log_n - 30))); return ZK_ERR_INVALID; }
    if (mode < 0 || mode > 3 || batch == 0 || batch > 65535) { zk_set_error("zk_ntt: bad mode/batch"); return ZK_ERR_INVALID; }
    ZK_TRY(zk_use_device(ctx));
    if (log_n == 0) return ZK_OK;     // size-1 transform is the identity (m^-1 = 1)
    NttSlot *t;
    ZK_TRY(get_tables(ctx, log_n, &t));
    const size_t n = (size_t)1 << log_n;
    const int inverse = (mode == ZK_NTT_IFFT || mode == ZK_NTT_ICOSET_FFT);
    const int coset_in = (mode == ZK_NTT_COSET_FFT);
    const int post = mode == ZK_NTT_IFFT ? 1 : (mode == ZK_NTT_ICOSET_FFT ? 2 : 0);
    if (!ctx->ntt_attr_done) {         // the attribute is per device; a context is bound to one device
        ZK_CUDA(cudaFuncSetAttribute(k_ntt_cols, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 << MAX_TILE_LOG));
        ZK_CUDA(cudaFuncSetAttribute(k_ntt_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 << MAX_TILE_LOG));
        ctx->ntt_attr_done = true;
    }
    Fr *data = (Fr *)d_data;
    const Fr *W = t->w.as<Fr>(), *G = t->g.as<Fr>(), *GI = t->gi.as<Fr>(), *consts = t->consts.as<Fr>();
    cudaStream_t st = ctx->stream;
    auto cols = [&](const Fr *in, Fr *out, PassGeom g, unsigned by, int cin) {
        int l2 = (int)g.log_sub - g.l1;
        int cols_log = MAX_TILE_LOG - g.l1; if (cols_log > l2) cols_log = l2;
        dim3 grid((unsigned)(((size_t)1 << g.log_sub) >> (g.l1 + cols_log)), by);
        k_ntt_cols<<<grid, NTT_THREADS, (size_t)32 << (g.l1 + cols_log), st>>>(in, out, g, cols_log, W, G, cin, inverse);
    };
    auto rows = [&](const Fr *in, Fr *out, PassGeom g, unsigned by, int cin, int pst) {
        int l2 = (int)g.log_sub - g.l1;
        int rows_log = MAX_TILE_LOG - l2; if (rows_log > g.l1) rows_log = g.l1;
        dim3 grid((unsigned)(((size_t)1 << g.log_sub) >> (l2 + rows_log)), by);
        k_ntt_rows<<<grid, NTT_THREADS, (size_t)32 << (l2 + rows_log), st>>>(in, out, g, rows_log, W, G, GI, consts, cin, inverse, pst);
    };
    if (log_n <= (unsigned)MAX_TILE_LOG) {
        PassGeom g{log_n, log_n, 0, 0, 0, 0};
        rows(data, data, g, (unsigned)batch, coset_in, post);              // whole vector in one tile: in place is safe
    } else if (log_n <= 2 * (unsigned)MAX_TILE_LOG) {
        ZK_TRY(ctx->ntt_tmp.reserve(n * 32 * batch));
        Fr *tmp = ctx->ntt_tmp.as<Fr>();
        PassGeom g{log_n, log_n, (int)log_n / 2, 0, 0, 0};
        cols(data, tmp, g, (unsigned)batch, coset_in);
        rows(tmp, data, g, (unsigned)batch, 0, post);
    } else {
        ZK_TRY(ctx->ntt_tmp.reserve(n * 32));
        Fr *tmp = ctx->ntt_tmp.as<Fr>();
        const int l0 = (int)log_n - 2 * MAX_TILE_LOG;                       // outer dimension 2^l0 <= 2^10
        PassGeom g0{log_n, log_n, l0, 0, 0, 0};
        PassGeom g1{log_n, 2 * MAX_TILE_LOG, MAX_TILE_LOG, l0, 1, l0};
        for (size_t b = 0; b < batch; b++) {                                // in stream order: vector b + 1 reuses tmp after b is done
            Fr *v = data + b * n;
            cols(v, tmp, g0, 1, coset_in);                                  // outer columns, twiddle w^(n' m0)
            cols(tmp, tmp, g1, 1u << l0, 0);                                // every row: inner columns (in place)
            rows(tmp, v, g1, 1u << l0, 0, post);                            // every row: inner rows, store at m0 + 2^l0 * m'
        }
    }
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_ntt_fr_device(zk_ctx *ctx, void *d_data, unsigned log_n, int mode) {
    if (!ctx || !d_data) { zk_set_error("zk_ntt_fr_device: NULL argument"); return ZK_ERR_INVALID; }
    return zk_ntt_run(ctx, d_data, log_n, mode, 1);
}
extern "C" int zk_ntt_fr(zk_ctx *ctx, uint64_t *data, unsigned log_n, int mode) {
    if (!ctx || !data) { zk_set_error("zk_ntt_fr: NULL argument"); return ZK_ERR_INVALID; }
    if (log_n > 32) { zk_set_error("PolynomialDegreeTooLarge: log_n = %u", log_n); return ZK_ERR_POLY_DEGREE_TOO_LARGE; }
    ZK_TRY(zk_use_device(ctx));
    size_t bytes = ((size_t)1 << log_n) * 32;
    ZK_TRY(ctx->stage_a.reserve(bytes));
    ZK_CUDA(cudaMemcpyAsync(ctx->stage_a.p, data, bytes, cudaMemcpyHostToDevice, ctx->stream));
    ZK_TRY(zk_ntt_run(ctx, ctx->stage_a.p, log_n, mode, 1));
    ZK_CUDA(cudaMemcpyAsync(data, ctx->stage_a.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

// ---- element-wise Fr kernels of create_proof (SURVEY.md §3.2) ------------------------------------------
namespace {
// evals: [batch][n_c] canonical -> dst[batch][which][m] Montgomery, zero padded (EvaluationDomain::from_coeffs)
__global__ void k_load_evals(const Fr *__restrict__ src, size_t n_c, unsigned log_m, int which, Fr *__restrict__ dst, int *err) {
    size_t m = (size_t)1 << log_m;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t b = blockIdx.y;
    if (i >= m) return;
    Fr v = Fr::zero();
    if (i < n_c) {
        Fr c = load_fr(src + b * n_c + i);
        if (!Fr::canonical_lt_mod(c)) atomicExch(err, 1);
        v = Fr::from_canonical(c);
    }
    store_fr(dst + ((b * 3 + which) << log_m) + i, v);
}
// h[b][i] = (a*b - c) * zinv   over the coset evaluations (mul_assign, sub_assign, divide_by_z_on_coset)
__global__ void k_quotient(const Fr *__restrict__ abc, unsigned log_m, const Fr *__restrict__ consts, Fr *__restrict__ h) {
    size_t m = (size_t)1 << log_m;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t b = blockIdx.y;
    if (i >= m) return;
    const Fr *base = abc + ((b * 3) << log_m);
    Fr a = load_fr(base + i), bb = load_fr(base + m + i), c = load_fr(base + 2 * m + i);
    store_fr(h + (b << log_m) + i, (a * bb - c) * load_fr(consts + 1));
}
// scal[b][i] = into_repr(h[b][i]), i < n_out; scal[b][n_out .. n_total) left for the caller (extra terms)
__global__ void k_into_repr(const Fr *__restrict__ h, unsigned log_m, size_t n_out, size_t n_total, Fr *__restrict__ scal) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t b = blockIdx.y;
    if (i >= n_out) return;
    store_fr(scal + b * n_total + i, load_fr(h + (b << log_m) + i).to_canonical());
}
// per proof: out[b][0] = 1, out[b][1] = r, out[b][2] = s, out[b][3] = -(r*s)  (all canonical) — the extra MSM terms
__global__ void k_blinding_terms(const Fr *__restrict__ r, const Fr *__restrict__ s, size_t batch, Fr *__restrict__ out, int *err) {
    size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    Fr rc = load_fr(r + b), sc = load_fr(s + b);
    if (!Fr::canonical_lt_mod(rc) || !Fr::canonical_lt_mod(sc)) atomicExch(err, 1);
    Fr one = Fr::zero(); one.l[0] = 1;
    Fr rs = (Fr::from_canonical(rc) * Fr::from_canonical(sc)).neg().to_canonical();
    store_fr(out + b * 4, one); store_fr(out + b * 4 + 1, rc); store_fr(out + b * 4 + 2, sc); store_fr(out + b * 4 + 3, rs);
}
// z[b][v] = from_repr(inputs | aux) for the R1CS evaluation
__global__ void k_witness_to_mont(const Fr *__restrict__ inputs, size_t n_in, const Fr *__restrict__ aux, size_t n_aux, Fr *__restrict__ z, int *err) {
    size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y, nv = n_in + n_aux;
    if (v >= nv) return;
    Fr c = v < n_in ? load_fr(inputs + b * n_in + v) : load_fr(aux + b * n_aux + (v - n_in));
    if (!Fr::canonical_lt_mod(c)) atomicExch(err, 1);
    store_fr(z + b * nv + v, Fr::from_canonical(c));
}
// dst[b][which][i] = <M_i, z_b> for i < n_c (CSR row i of the matrix `which`), the appended `input_i * 0 = 0` rows for
// n_c <= i < n_c + n_in (A only: the input's value), zero padding up to m.  What ProvingAssignment::enforce computes on
// the host in bellman (SURVEY.md §3.2), moved to the device for a fixed constraint system (SURVEY.md §8 f4).
__global__ void k_r1cs_eval(const uint32_t *__restrict__ row_ptr, const uint32_t *__restrict__ col, const Fr *__restrict__ coeff,
                            const Fr *__restrict__ z, size_t n_c, size_t n_in, size_t nv, unsigned log_m, int which, Fr *__restrict__ dst) {
    size_t m = (size_t)1 << log_m;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= m) return;
    const Fr *zb = z + b * nv;
    Fr acc = Fr::zero();
    if (i < n_c) {
        for (uint32_t k = row_ptr[i]; k < row_ptr[i + 1]; k++) acc = acc + load_fr(coeff + k) * load_fr(zb + col[k]);
    } else if (which == 0 && i < n_c + n_in) acc = load_fr(zb + (i - n_c));
    store_fr(dst + ((b * 3 + which) << log_m) + i, acc);
}
// coefficients canonical -> Montgomery (once, at zk_r1cs_load)
__global__ void k_fr_to_mont(const Fr *__restrict__ in, size_t n, Fr *__restrict__ out, int *err) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr c = load_fr(in + i);
    if (!Fr::canonical_lt_mod(c)) atomicExch(err, 1);
    store_fr(out + i, Fr::from_canonical(c));
}
}  // namespace

int zk_fr_to_mont(zk_ctx *ctx, const void *d_in, size_t n, void *d_out) {
    if (n) k_fr_to_mont<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>((const Fr *)d_in, n, (Fr *)d_out, ctx->d_err);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
int zk_fr_witness_to_mont(zk_ctx *ctx, const void *d_inputs, size_t n_in, const void *d_aux, size_t n_aux, size_t batch, void *d_z) {
    size_t nv = n_in + n_aux;
    k_witness_to_mont<<<dim3((unsigned)((nv + 255) / 256), (unsigned)batch), 256, 0, ctx->stream>>>((const Fr *)d_inputs, n_in, (const Fr *)d_aux, n_aux, (Fr *)d_z, ctx->d_err);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
int zk_fr_r1cs_eval(zk_ctx *ctx, const uint32_t *d_row_ptr, const uint32_t *d_col, const void *d_coeff, const void *d_z, size_t n_c, size_t n_in,
                    size_t nv, unsigned log_m, int which, size_t batch, void *d_dst) {
    size_t m = (size_t)1 << log_m;
    k_r1cs_eval<<<dim3((unsigned)((m + 127) / 128), (unsigned)batch), 128, 0, ctx->stream>>>(d_row_ptr, d_col, (const Fr *)d_coeff, (const Fr *)d_z, n_c, n_in, nv,
                                                                                          log_m, which, (Fr *)d_dst);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

int zk_fr_load_evals(zk_ctx *ctx, const void *d_src, size_t n_c, unsigned log_m, int which, size_t batch, void *d_dst) {
    size_t m = (size_t)1 << log_m;
    k_load_evals<<<dim3((unsigned)((m + 255) / 256), (unsigned)batch), 256, 0, ctx->stream>>>((const Fr *)d_src, n_c, log_m, which, (Fr *)d_dst, ctx->d_err);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
int zk_fr_quotient(zk_ctx *ctx, const void *d_abc, unsigned log_m, size_t batch, void *d_h) {
    NttSlot *t;
    ZK_TRY(get_tables(ctx, log_m, &t));
    size_t m = (size_t)1 << log_m;
    k_quotient<<<dim3((unsigned)((m + 255) / 256), (unsigned)batch), 256, 0, ctx->stream>>>((const Fr *)d_abc, log_m, t->consts.as<Fr>(), (Fr *)d_h);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
int zk_fr_into_repr(zk_ctx *ctx, const void *d_h, unsigned log_m, size_t n_out, size_t n_total, size_t batch, void *d_scal) {
    k_into_repr<<<dim3((unsigned)((n_out + 255) / 256), (unsigned)batch), 256, 0, ctx->stream>>>((const Fr *)d_h, log_m, n_out, n_total, (Fr *)d_scal);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
int zk_fr_blinding_terms(zk_ctx *ctx, const void *d_r, const void *d_s, size_t batch, void *d_out) {
    k_blinding_terms<<<(unsigned)((batch + 63) / 64), 64, 0, ctx->stream>>>((const Fr *)d_r, (const Fr *)d_s, batch, (Fr *)d_out, ctx->d_err);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
