// Shared host-side declarations of libzkb200 (not part of the public ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <type_traits>
#include <vector>
#include "../../include/zkb200.h"

void zk_set_error(const char *fmt, ...);
#define ZK_CUDA(call)                                                                                  \
    do {                                                                                               \
        cudaError_t e__ = (call);                                                                      \
        if (e__ != cudaSuccess) {                                                                      \
            zk_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));       \
            return ZK_ERR_CUDA;                                                                        \
        }                                                                                              \
    } while (0)
#define ZK_TRY(call) do { int r__ = (call); if (r__ != ZK_OK) return r__; } while (0)

// grow-only device buffer
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    int reserve(size_t bytes) {
        if (bytes <= cap) return ZK_OK;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + (bytes >> 3) + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { zk_set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e)); return ZK_ERR_CUDA; }
        cap = want;
        return ZK_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

// carves a workspace out of one grow-only buffer, 256-byte aligned pieces (base NULL: only sums the size)
struct Carve {
    uint8_t *base = nullptr;
    size_t off = 0;
    template <class T> T *take(size_t count) {
        T *p = reinterpret_cast<T *>(base ? base + off : nullptr);
        off += (count * sizeof(T) + 255) & ~(size_t)255;
        return p;
    }
};

// one cached set of NTT twiddle tables (ntt.cu)
struct NttSlot { unsigned log_n = 0; bool valid = false; uint64_t last_use = 0; DevBuf w, g, gi, consts; };

// tuning options of a context (zk_ctx_set_opt); the prover lanes inherit them
struct zk_opts {
    long ba_min_entries = 1l << 22;    // ZK_OPT_AFFINE_MIN_ENTRIES; -1 = batched-affine rounds off
    long ba_levels = -1;               // ZK_OPT_AFFINE_LEVELS (-1 = from the average bucket length)
    long verify_lanes = 1;             // ZK_OPT_VERIFY_LANES: 1 = lane-parallel Miller loop / final exponentiation, 0 = thread per proof
};

struct zk_ctx {
    zk_opts opts;
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 0;
    int *d_err = nullptr;          // device error flag (non-canonical scalar etc.)
    // MSM workspace
    DevBuf aff_pts0, aff_pts1, aff_scratch, aff_off0, aff_off1, aff_sizes0, aff_sizes1, aff_tot;   // batched-affine rounds (msm_batchaff.cuh)
    DevBuf scalars, digits, tile_hist, tile_off, sizes, bucket_off, task_off, scan_scratch, sorted, partials, buckets, red_part, red_x, red_rows, sorted2, coarse_off, coarse_sizes, task_order, len_hist, heavy_list, red_tmp, result, out_bytes;
    bool len_hist_zeroed = false;
    // generic staging
    DevBuf stage_a, stage_b, stage_c;
    // NTT workspace + twiddle tables (per context: ordered on this context's stream, freed with it)
    DevBuf ntt_tmp;
    NttSlot ntt_slots[4];
    uint64_t ntt_clock = 0;
    bool ntt_attr_done = false;
    // groth16 workspace
    DevBuf g_a, g_b, g_c, g_h, g_scal, g_misc;
    // verifier workspace (pairing.cu)
    DevBuf v_pts, v_stat, v_coef, v_f, v_part;
    DevBuf v_jj;                   // zk_groth16_verify_points_batch: decoded public inputs and per-point status (jubjub.cu)
    // zk_elgamal_decrypt_batch (elgamal.cu): the encodings of i P_G for i < 10^6 and their index, built by the first call
    DevBuf eg_table, eg_index;
    bool eg_ready = false;
    DevBuf bal;                    // zk_balances_confidential_block (balances.cu), zk_balances_anonymous_block
                                   // (anon_balances.cu) and zk_assets_block (assets.cu): workspace
    DevBuf imp;                    // zk_import_confidential_block / zk_import_assets_block (import.cu): round buffers
    DevBuf io;                     // the host forms' arrays (Stage); no device form reads it, and every host form
                                   // synchronises before it returns, so one buffer serves them all
    DevBuf imp_as;                 // zk_import_asset_calls (import.cu): the hash table, references and grown slot table
    DevBuf tb;                     // zk_confidential_fields_batch (tx_build.cu): the g_epoch window table and the rows' points
    DevBuf hd;                     // zk_xsk_derive_batch / zk_xpgk_derive_batch (hd_keys.cu): each named parent's pgk and tag
    DevBuf jm;                     // zk_jubjub_msm / zk_redjubjub_batch_verify (jubjub_msm.cu): bases, scalars, sort and buckets
    // live kernel timing (zk_ctx_profile): CUDA events around the dominant kernel on ctx->stream
    bool prof_on = false;
    std::vector<cudaEvent_t> prof_events;   // pairs (start, stop)
    zk_ctx *aux2 = nullptr;        // third lane: the A MSM and s * g_a (independent of the NTT chain)
    zk_ctx *aux3 = nullptr;        // fourth lane: the B1 MSM and r * g_b1
    DevBuf g_scal3;                // A-query scalars
    zk_ctx *aux = nullptr;         // second lane (own stream + workspace) on the same device: the prover's G2 MSM overlaps the G1 work
    DevBuf g_scal2;                // B-query scalars (shared by the G1 and G2 B MSMs)
    // asynchronous MSM (zk_msm_begin / zk_msm_end): everything after the bucket accumulation runs on a HIGH-PRIORITY stream, so that
    // with two contexts in flight the latency-bound tail of one MSM is scheduled ahead of the other's accumulation blocks
    cudaStream_t tail = nullptr;
    cudaEvent_t ev_front = nullptr, ev_tail = nullptr;
    bool split_tail = false;       // set by zk_msm_*begin around the driver call
    size_t pending_bytes = 0;      // result bytes of the MSM in flight (0 = none)
    uint8_t *h_pinned = nullptr;   // small pinned buffer for results
    size_t h_pinned_cap = 0;
};

// A host form's staging through ctx->io.  Each array is registered once: its host pointer, the device pointer to fill in,
// its element count and its direction.  up() carves ctx->io in Carve's pieces, fills in every device pointer and copies
// the in and in-out arrays up; down(), after the caller has enqueued its run, copies the out and in-out arrays back.  Both
// enqueue on ctx->stream and neither synchronises.  A NULL host pointer gets a NULL device pointer, no space and no
// copy; a count of 0 gets a valid device pointer and no copy.  An output registered with rows and width comes down for
// *rows rows of width elements (*rows read by down(), at most count elements): a table whose final size is known only
// after the run.
struct Stage {
    template <class T, class D> void in(const T *h, D *&d, size_t count) { add(h, d, count, true, false, nullptr, 1); }
    template <class T, class D> void out(T *h, D *&d, size_t count, const size_t *rows = nullptr, size_t width = 1) {
        add(h, d, count, false, true, rows, width);
    }
    template <class T, class D> void inout(T *h, D *&d, size_t count) { add(h, d, count, true, true, nullptr, 1); }

    int up(zk_ctx *ctx) {
        Carve sizing;
        for (const Item &it : items) sizing.take<uint8_t>(it.elem * it.count);
        ZK_TRY(ctx->io.reserve(sizing.off ? sizing.off : 1));     // 1: a buffer to point into when every count is 0
        Carve c{ctx->io.as<uint8_t>(), 0};
        for (Item &it : items) {
            it.dev = c.take<uint8_t>(it.elem * it.count);
            it.set(it.slot, it.dev);
            if (it.to_dev && it.count) ZK_CUDA(cudaMemcpyAsync(it.dev, it.host, it.elem * it.count, cudaMemcpyHostToDevice, ctx->stream));
        }
        return ZK_OK;
    }
    int down(zk_ctx *ctx) {
        for (const Item &it : items) {
            const size_t n = it.rows && *it.rows * it.width < it.count ? *it.rows * it.width : it.count;
            if (it.to_host && n) ZK_CUDA(cudaMemcpyAsync(it.host, it.dev, it.elem * n, cudaMemcpyDeviceToHost, ctx->stream));
        }
        return ZK_OK;
    }

  private:
    struct Item {
        void *host, *slot;
        void (*set)(void *slot, uint8_t *dev);
        uint8_t *dev;
        size_t elem, count, width;
        bool to_dev, to_host;
        const size_t *rows;
    };
    std::vector<Item> items;
    template <class T, class D> void add(const T *h, D *&d, size_t count, bool to_dev, bool to_host, const size_t *rows, size_t width) {
        static_assert(std::is_same<typename std::remove_const<D>::type, T>::value, "a host array and its device copy have one element type");
        d = nullptr;
        if (h)
            items.push_back({const_cast<T *>(h), &d, [](void *slot, uint8_t *dev) { *static_cast<D **>(slot) = reinterpret_cast<D *>(dev); },
                             nullptr, sizeof(T), count, width, to_dev, to_host, rows});
    }
};

struct zk_bases {
    int group = 1;       // 1 = G1, 2 = G2
    int device = 0;
    size_t n = 0;        // bases (table row stride)
    int c = 0, W = 0;
    bool tables = false;
    void *d_tbl = nullptr;   // [W or 1][n] affine
};

int zk_use_device(zk_ctx *ctx);
// internal MSM driver: result XYZZ points (one per batch item) left in ctx->result (device)
int zk_msm_run(zk_ctx *ctx, const zk_bases *b, const void *d_scalars, size_t n, size_t batch);
int zk_encode_results(zk_ctx *ctx, int group, size_t count, int compressed, uint8_t *out_host);

// hot-TU entry points (msm_hot.cu)
int zk_msm_run_g1(zk_ctx *ctx, const zk_bases *b, const uint32_t *d_scalars, size_t n, size_t batch);
int zk_build_tables_g1(zk_ctx *ctx, zk_bases *b);
int zk_encode_results_g1(zk_ctx *ctx, size_t count, int compressed, uint8_t *d_out);
void zk_launch_bench_modmul(int field, int blocks, int threads, int iters, void *sink, cudaStream_t st);
int zk_bases_from_device(zk_ctx *ctx, int group, const void *d_points, size_t n, int window_bits, int precompute, zk_bases **out);
int zk_ntt_run(zk_ctx *ctx, void *d_data, unsigned log_n, int mode, size_t batch);
int zk_fr_load_evals(zk_ctx *ctx, const void *d_src, size_t n_c, unsigned log_m, int which, size_t batch, void *d_dst);
int zk_fr_quotient(zk_ctx *ctx, const void *d_abc, unsigned log_m, size_t batch, void *d_h);
int zk_fr_into_repr(zk_ctx *ctx, const void *d_h, unsigned log_m, size_t n_out, size_t n_total, size_t batch, void *d_scal);
int zk_fr_blinding_terms(zk_ctx *ctx, const void *d_r, const void *d_s, size_t batch, void *d_out);
int zk_check_err_flag(zk_ctx *ctx);
// d_err[ZK_ERR_SLOT_ACCOUNT]: ~(the lowest account whose stored ciphertext failed to read) in zk_balances_confidential_block
// and zk_balances_anonymous_block (the lowest slot in zk_assets_block), 0: none
constexpr int ZK_ERR_SLOT_ACCOUNT = 2;
// balances.cu's passes over a block's elements, shared with anon_balances.cu, enqueued on ctx->stream:
//   zk_bal_sort  stable LSD radix sort of ne keys (each <= 2 n_acct; keys0 holds them, keys1 / vals0 / vals1 / hist /
//                totals are workspace of balances.cuh's sizes) with the element ids; *keys / *vals: the sorted pair
//   zk_bal_scan  segmented exclusive scan of delta[vals[j]] in key order over L levels (lvl_n[0] = ne; level l >= 1 has
//                lvl_n[l] items and its lvl_agg / lvl_out / lvl_head; lvl_out[0] receives the scan, lvl_head[0] the heads)
//   zk_bal_prefix_sum  exclusive prefix sum of n > 0 uint32 counters in place (totals: 1024 words of workspace); also
//                serves assets.cu, which numbers its segments with it
namespace zkbal { struct Pair; }
int zk_bal_prefix_sum(zk_ctx *ctx, uint32_t *c, size_t n, uint32_t *totals);
int zk_bal_sort(zk_ctx *ctx, size_t ne, size_t n_acct, uint32_t *keys0, uint32_t *keys1, uint32_t *vals0, uint32_t *vals1, uint32_t *hist,
                uint32_t *totals, const uint32_t **keys, const uint32_t **vals);
int zk_bal_scan(zk_ctx *ctx, const uint32_t *keys, const uint32_t *vals, const zkbal::Pair *delta, size_t L, const size_t *lvl_n,
                zkbal::Pair *const *lvl_agg, zkbal::Pair *const *lvl_out, uint8_t *const *lvl_head);
// lane-parallel verifier kernels (pairing_lanes.cu)
void zk_launch_miller_lanes(cudaStream_t st, size_t n, const void *a, const void *acc, const void *c, const void *coef_b, const void *gamma, int gamma_inf,
                            const void *delta, int delta_inf, const uint8_t *status, void *f);
void zk_launch_verify_final_lanes(cudaStream_t st, size_t n, const void *f, const void *alpha_beta, const uint8_t *status, uint8_t *verdict);
// Jubjub public-input decoding (jubjub.cu): xy[2 p], xy[2 p + 1] = canonical x, y of encoding p, status[p] 0..3; then verdict
// ZK_VERDICT_INPUT_REJECTED for every transaction i with a nonzero status[i * n_points + j]
constexpr uint8_t ZK_VERDICT_INPUT_REJECTED = 4;
void zk_launch_jubjub_into_xy(cudaStream_t st, const uint8_t *d_enc, size_t n, uint64_t *d_xy, uint8_t *d_status);
void zk_launch_mark_rejected_inputs(cudaStream_t st, size_t n, size_t n_points, const uint8_t *d_status, uint8_t *d_verdicts);
int zk_fr_to_mont(zk_ctx *ctx, const void *d_in, size_t n, void *d_out);
int zk_fr_witness_to_mont(zk_ctx *ctx, const void *d_inputs, size_t n_in, const void *d_aux, size_t n_aux, size_t batch, void *d_z);
int zk_fr_r1cs_eval(zk_ctx *ctx, const uint32_t *d_row_ptr, const uint32_t *d_col, const void *d_coeff, const void *d_z, size_t n_c, size_t n_in,
                    size_t nv, unsigned log_m, int which, size_t batch, void *d_dst);
