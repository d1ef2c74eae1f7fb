// Host-side MSM driver, templated on the base field so that G1 is compiled in the hot translation unit
// (msm_hot.cu, everything inlined) and G2 in the cold one (engine.cu).  See msm.cuh for the schedule.
#pragma once
#include "internal.h"
#include "msm.cuh"
#include "msm_batchaff.cuh"
#include "codec.cuh"
#include <stdlib.h>

namespace zkmsm {

template <class F>
int build_tables_t(zk_ctx *ctx, zk_bases *b) {
    unsigned thr = 128, blk = (unsigned)((b->n + thr * PRE_K - 1) / (thr * PRE_K));
    k_precompute<F><<<blk, thr, 0, ctx->stream>>>((Affine<F> *)b->d_tbl, (uint32_t)b->n, b->c, b->W);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

template <class F>
int msm_run_t(zk_ctx *ctx, const zk_bases *b, const uint32_t *d_scalars, size_t n, size_t batch) {
    cudaStream_t st = ctx->stream;
    const int c = b->c, W = b->W, nbins = 1 << (c - 1);
    // sort domains: with tables one domain per batch item holding all W windows; without tables one per window
    const bool tables = b->tables;
    if (!tables && batch != 1) { zk_set_error("batched MSM needs precomputed tables"); return ZK_ERR_INVALID; }
    const size_t n_dom = tables ? batch : (size_t)W;
    const uint64_t e_dom = tables ? (uint64_t)n * W : (uint64_t)n;
    const size_t E = (size_t)n * W * batch;
    if (E >= ((size_t)1 << 31)) { zk_set_error("MSM too large for 31-bit entry payloads (n*W*batch = %zu)", E); return ZK_ERR_INVALID; }
    // sort tiles: fixed TILE for the one-level sort (c <= 16, up to 128 KB of shared counters per block); the coarse level of
    // the two-level sort (c > 16, 2 KB of counters) uses small tiles, enough of them to fill every SM twice
    const bool two_level = c > 16;
    const int low = two_level ? (c - 1) - 9 : 0, sort_bins = two_level ? 512 : nbins;
    size_t smem = (size_t)sort_bins * 4;
    uint32_t tile_len = TILE;
    if (two_level) {
        int per_sm = 0;
        ZK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_coarse_scatter, COARSE_THREADS, 0));
        tile_len = coarse_tile_len(e_dom, n_dom, per_sm * ctx->sm_count);
    }
    const int tiles = (int)((e_dom + tile_len - 1) / tile_len);
    const size_t NB = n_dom * nbins;
    // tasks: round(size_b / task_len) >= 1 per non-empty bucket, summed <= total/task_len + NB (k_pick_task_len), and
    // total/task_len <= E/TASK_LEN_MAX + two waves of k_accumulate (sm_count x 384 resident tasks; 1024 per SM leaves margin)
    size_t t_max = E / TASK_LEN_MAX + 2 * (size_t)ctx->sm_count * 1024u + 1;
    t_max += NB + 1;
    const size_t pt = sizeof(XYZZ<F>);
    ZK_TRY(ctx->digits.reserve(E * 4));
    ZK_TRY(ctx->tile_hist.reserve(n_dom * tiles * (size_t)(c > 16 ? 512 : nbins) * 4));
    ZK_TRY(ctx->tile_off.reserve(n_dom * tiles * (size_t)(c > 16 ? 512 : nbins) * 4));
    ZK_TRY(ctx->sizes.reserve((NB + 1) * 4));
    ZK_TRY(ctx->bucket_off.reserve((NB + 1) * 4));
    ZK_TRY(ctx->task_off.reserve((NB + 1) * 4));
    ZK_TRY(ctx->scan_scratch.reserve((2 * (NB / SCAN_B + 8) + 4096) * 4));
    ZK_TRY(ctx->sorted.reserve(E * 4));
    ZK_TRY(ctx->partials.reserve(t_max * pt));
    ZK_TRY(ctx->buckets.reserve(NB * pt));
    const int n_bits = c;                      // digit values d in [1, 2^(c-1)] need c bits
    const int n_slices = (nbins / 2 + RED_SLICE / 2 - 1) / (RED_SLICE / 2) > 0 ? (nbins / 2 + RED_SLICE / 2 - 1) / (RED_SLICE / 2) : 1;   // slices of RED_SLICE/2 qualifying digit values
    ZK_TRY(ctx->red_part.reserve(2 * n_dom * n_bits * (size_t)n_slices * pt));      // x2: the row/column scheme runs 2 pseudo-domains per domain
    ZK_TRY(ctx->red_x.reserve(2 * n_dom * n_bits * pt));
    ZK_TRY(ctx->result.reserve((n_dom + batch + 1) * pt));

    uint32_t *digits = ctx->digits.as<uint32_t>();
    {   // 1. digits: grid.y = batch item, layout [batch][W][n]
        dim3 g((unsigned)((n + 255) / 256), (unsigned)batch);
        k_msm_digits<<<g, 256, 0, st>>>(d_scalars, (uint32_t)n, c, W, digits, ctx->d_err);
    }
    // 2. counting sort per domain.  Up to 16-bit windows the 2^(c-1) bucket counters fit in shared memory (one level);
    //    wider windows sort by the high 9 key bits first and finish each coarse bin in shared memory (k_fine_sort).
    const size_t SB = n_dom * (size_t)sort_bins;
    if (smem > 48 * 1024) {
        ZK_CUDA(cudaFuncSetAttribute(k_tile_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ZK_CUDA(cudaFuncSetAttribute(k_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    dim3 gs((unsigned)tiles, (unsigned)n_dom);
    if (!two_level) {
        k_tile_hist<<<gs, SORT_THREADS, smem, st>>>(digits, e_dom, nbins, 0, ctx->tile_hist.as<uint32_t>(), tiles, tile_len, false);
        k_col_scan<<<(unsigned)((NB + 255) / 256), 256, 0, st>>>(ctx->tile_hist.as<uint32_t>(), ctx->tile_off.as<uint32_t>(), ctx->sizes.as<uint32_t>(),
                                                                nbins, tiles, (int)n_dom);
        exclusive_scan<false>(ctx->sizes.as<uint32_t>(), ctx->bucket_off.as<uint32_t>(), NB, ctx->scan_scratch.as<uint32_t>(), st);
        k_scatter<<<gs, SORT_THREADS, smem, st>>>(digits, e_dom, nbins, ctx->tile_off.as<uint32_t>(), ctx->bucket_off.as<uint32_t>(),
                                                  ctx->sorted.as<uint32_t>(), tiles, tile_len);
    } else {
        ZK_TRY(ctx->sorted2.reserve(E * sizeof(uint2)));           // {entry, bucket key} per entry (k_coarse_scatter)
        ZK_TRY(ctx->coarse_off.reserve((SB + 1) * 4)); ZK_TRY(ctx->coarse_sizes.reserve((SB + 1) * 4));
        // per-tile counters bin-major ([domain][bin][tile]): k_bin_scan reads each bin's counters contiguously
        k_tile_hist<<<gs, COARSE_THREADS, smem, st>>>(digits, e_dom, sort_bins, low, ctx->tile_hist.as<uint32_t>(), tiles, tile_len, true);
        k_bin_scan<<<(unsigned)SB, COARSE_THREADS, 0, st>>>(ctx->tile_hist.as<uint32_t>(), ctx->tile_off.as<uint32_t>(), ctx->coarse_sizes.as<uint32_t>(), tiles);
        exclusive_scan<false>(ctx->coarse_sizes.as<uint32_t>(), ctx->coarse_off.as<uint32_t>(), SB, ctx->scan_scratch.as<uint32_t>(), st);
        k_coarse_scatter<<<gs, COARSE_THREADS, 0, st>>>(digits, e_dom, low, ctx->tile_off.as<uint32_t>(), ctx->coarse_off.as<uint32_t>(),
                                                        ctx->sorted2.as<uint2>(), tiles, tile_len);
        ZK_CUDA(cudaFuncSetAttribute(k_fine_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, FINE_STAGE * 4));
        k_fine_sort<<<dim3(512, (unsigned)n_dom), 1024, FINE_STAGE * 4, st>>>(ctx->sorted2.as<uint2>(), ctx->coarse_off.as<uint32_t>(), 512, low,
                                                                 ctx->sizes.as<uint32_t>(), ctx->bucket_off.as<uint32_t>(), ctx->sorted.as<uint32_t>());
    }
    // 2b. batched-affine rounds (msm_batchaff.cuh): each round halves every bucket at ~6.4 products per addition instead of the 10
    //     of an XYZZ mixed addition, with ONE shared field inversion per round.  The rounds pay off in throughput (several MSMs in
    //     flight, batched proving) but each adds the latency of its serial inversion, so only MSMs with >= 2^22 entries take them
    //     (zk_ctx_set_opt), and the
    //     number of rounds follows the average bucket length (the host knows the upper bound E / NB; sparse scalars make the
    //     rounds cheaper, not wrong).
    // the points of the next pass: the window tables (rows x | y), then each round's outputs as an x plane and a y plane
    const F *cur_x = (const F *)b->d_tbl, *cur_y = nullptr;
    const uint32_t *cur_sorted = ctx->sorted.as<uint32_t>(), *cur_off = ctx->bucket_off.as<uint32_t>(), *cur_sizes = ctx->sizes.as<uint32_t>();
    // zk_ctx_profile: the bucket-accumulation stage (affine rounds, if any, + the XYZZ pass); destroyed here unless handed to the context
    struct ProfPair {
        cudaEvent_t a = nullptr, b = nullptr; bool kept = false;
        ~ProfPair() { if (!kept) { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); } }
    } prof;
    cudaEvent_t &ev0 = prof.a, &ev1 = prof.b;
    {
        int levels = 0;
        if (ctx->opts.ba_min_entries >= 0 && (long)E >= ctx->opts.ba_min_entries) {      // small MSMs stay on the XYZZ pass alone (see above)
            if (ctx->opts.ba_levels >= 0) levels = (int)(ctx->opts.ba_levels < BA_MAX_LEVELS ? ctx->opts.ba_levels : BA_MAX_LEVELS);
            else for (size_t avg = E / NB; avg >= 12 && levels < BA_MAX_LEVELS; avg >>= 1) levels++;      // 26 per bucket -> 2 rounds, 76 -> 3
        }
        if (ctx->prof_on && levels > 0) { cudaEventCreate(&ev0); cudaEventCreate(&ev1); cudaEventRecord(ev0, st); }
        size_t in_max = E;
        int minb = BA_MINB, k_force = 0;
        (void)minb;
#ifdef ZK_EXPERIMENTS
        if (const char *e = getenv("ZK_BA_MINB")) minb = atoi(e);
        if (const char *e = getenv("ZK_BA_K")) k_force = atoi(e);
#endif
        DevBuf *pts_buf[2] = {&ctx->aff_pts0, &ctx->aff_pts1}, *off_buf[2] = {&ctx->aff_off0, &ctx->aff_off1}, *sz_buf[2] = {&ctx->aff_sizes0, &ctx->aff_sizes1};
        if (levels > 0) {
            if (ba_smem_backward<F>() > 48 * 1024) {
                ZK_CUDA(cudaFuncSetAttribute(k_ba_backward<F, true, BA_MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba_smem_backward<F>()));
                ZK_CUDA(cudaFuncSetAttribute(k_ba_backward<F, false, BA_MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba_smem_backward<F>()));
#ifdef ZK_EXPERIMENTS
                ZK_CUDA(cudaFuncSetAttribute(k_ba_backward<F, true, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba_smem_backward<F>()));
                ZK_CUDA(cudaFuncSetAttribute(k_ba_backward<F, false, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba_smem_backward<F>()));
#endif
            }
            if (ba_smem_invert<F>() > 48 * 1024)
                ZK_CUDA(cudaFuncSetAttribute(k_ba_invert<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba_smem_invert<F>()));
        }
        for (int l = 0; l < levels; l++) {
            const size_t out_max = (in_max + NB) / 2 + 1;
            int K = BA_K;
            if (k_force > 0) K = k_force;
            const unsigned grid = (unsigned)((out_max + (size_t)BA_T * K - 1) / ((size_t)BA_T * K));
            const size_t T_total = (size_t)grid * BA_T;
            DevBuf *pts_o = pts_buf[l & 1], *off_o = off_buf[l & 1], *sz_o = sz_buf[l & 1];
            ZK_TRY(pts_o->reserve(out_max * sizeof(Affine<F>)));
            F *out_x = pts_o->as<F>(), *out_y = out_x + out_max;        // x plane, then y plane
            ZK_TRY(off_o->reserve((NB + 1) * 4)); ZK_TRY(sz_o->reserve((NB + 1) * 4));
            ZK_TRY(ctx->aff_scratch.reserve((size_t)(K + 1) * T_total * sizeof(F)));
            const size_t n_tot = (size_t)grid * (BA_T / 32);            // one total per warp
            ZK_TRY(ctx->aff_tot.reserve(3 * n_tot * sizeof(F)));
            F *tot = ctx->aff_tot.as<F>(), *tot_scr = tot + n_tot, *tot_inv = tot + 2 * n_tot;
            k_half_sizes<<<(unsigned)((NB + 255) / 256), 256, 0, st>>>(cur_off, sz_o->as<uint32_t>(), (uint32_t)NB);
            exclusive_scan<false>(sz_o->as<uint32_t>(), off_o->as<uint32_t>(), NB, ctx->scan_scratch.as<uint32_t>(), st);
            const uint32_t *off_out = off_o->as<uint32_t>();
            if (l == 0)
                k_ba_forward<F, true><<<grid, BA_T, ba_smem_forward<F>(), st>>>(cur_x, cur_y, cur_sorted, cur_off, off_out, (uint32_t)NB, K, ctx->aff_scratch.as<F>(), tot);
            else
                k_ba_forward<F, false><<<grid, BA_T, ba_smem_forward<F>(), st>>>(cur_x, cur_y, nullptr, cur_off, off_out, (uint32_t)NB, K, ctx->aff_scratch.as<F>(), tot);
            k_ba_invert<F><<<1, BA_INV_T, ba_smem_invert<F>(), st>>>(tot, off_out, (uint32_t)NB, K, tot_scr, tot_inv);
            const int Kb = K;
#define ZK_BA_BWD(FIRST_, MB_) k_ba_backward<F, FIRST_, MB_><<<grid, BA_T, ba_smem_backward<F>(), st>>>(cur_x, cur_y, cur_sorted, cur_off, off_out, (uint32_t)NB, Kb, \
                                                                                                    ctx->aff_scratch.as<F>(), tot_inv, out_x, out_y)
#ifdef ZK_EXPERIMENTS
            if (minb == 3) { if (l == 0) ZK_BA_BWD(true, 3); else ZK_BA_BWD(false, 3); } else
#endif
            { if (l == 0) ZK_BA_BWD(true, BA_MINB); else ZK_BA_BWD(false, BA_MINB); }
#undef ZK_BA_BWD
            cur_x = out_x; cur_y = out_y; cur_sorted = nullptr;
            cur_off = off_out; cur_sizes = sz_o->as<uint32_t>();
            in_max = out_max;
        }
    }
    uint32_t *d_task_len = (uint32_t *)(ctx->d_err + 8);
    const uint32_t capacity = (uint32_t)ctx->sm_count * 3u * 128u;      // k_accumulate: 3 CTAs of 128 threads per SM
    unsigned long long *d_work = (unsigned long long *)(ctx->d_err + (sizeof(F) == sizeof(Fq) ? 10 : 12));   // G1 / G2 addition counters
    k_pick_task_len<<<1, 1, 0, st>>>(cur_off + NB, ctx->bucket_off.as<uint32_t>() + NB, d_task_len, capacity, d_work, d_work + 2);
    exclusive_scan<true>(cur_sizes, ctx->task_off.as<uint32_t>(), NB, ctx->scan_scratch.as<uint32_t>(), st, d_task_len);
    // 3. accumulate + combine.  The payload of an entry is its position in the domain = [w][i] index;
    //    with tables that is the table index when n == b->n (checked by the callers).
    XYZZ<F> *partials = ctx->partials.as<XYZZ<F>>(), *buckets = ctx->buckets.as<XYZZ<F>>();
    // task order by decreasing length when buckets are short and uneven (batched proving, wide windows); one large MSM with
    // 16-bit windows has ~equal tasks already and skips it
    const uint32_t *order = nullptr;
    {
        bool want = E / NB < 256;
        if (want) {
            ZK_TRY(ctx->task_order.reserve(t_max * 4)); ZK_TRY(ctx->len_hist.reserve(2 * LEN_BINS * 4 + 64));
            uint32_t *gh = ctx->len_hist.as<uint32_t>(), *cur = gh + LEN_BINS;
            if (!ctx->len_hist_zeroed) { ZK_CUDA(cudaMemsetAsync(gh, 0, 2 * LEN_BINS * 4, st)); ctx->len_hist_zeroed = true; }
            unsigned nb = (unsigned)((NB + LEN_BLOCK - 1) / LEN_BLOCK);
            k_len_hist<<<nb, LEN_BLOCK, 0, st>>>(cur_off, ctx->task_off.as<uint32_t>(), (uint32_t)NB, gh);
            k_len_scan<<<1, LEN_BINS, 0, st>>>(gh, cur);
            k_len_place<<<nb, LEN_BLOCK, 0, st>>>(cur_off, ctx->task_off.as<uint32_t>(), (uint32_t)NB, cur, ctx->task_order.as<uint32_t>());
            order = ctx->task_order.as<uint32_t>();
        }
    }
    {
        const uint32_t *so = cur_sorted, *bo = cur_off, *to = ctx->task_off.as<uint32_t>();
        unsigned grid = (unsigned)((t_max + 127) / 128);
        if (ctx->prof_on && !ev0) { cudaEventCreate(&ev0); cudaEventCreate(&ev1); cudaEventRecord(ev0, st); }
        k_accumulate<F, 3><<<grid, 128, 0, st>>>(cur_x, cur_y, so, bo, to, (uint32_t)NB, order, partials);      // 3 CTAs / SM (168 registers, no spills)
    }
    if (ctx->prof_on) { cudaEventRecord(ev1, st); ctx->prof_events.push_back(ev0); ctx->prof_events.push_back(ev1); prof.kept = true; }
    if (ctx->split_tail) {             // asynchronous MSM: combine / reduction continue on the high-priority tail stream
        ZK_CUDA(cudaEventRecord(ctx->ev_front, st));
        ZK_CUDA(cudaStreamWaitEvent(ctx->tail, ctx->ev_front, 0));
        st = ctx->tail;
    }
    const size_t sm_warp = 4 * 32 * pt;      // 4 warps x 32 points
    if (sm_warp > 48 * 1024) {
        ZK_CUDA(cudaFuncSetAttribute(k_combine_warp<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_warp));
        ZK_CUDA(cudaFuncSetAttribute(k_bit_sums<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_warp));
        ZK_CUDA(cudaFuncSetAttribute(k_sum_points<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_warp));
        ZK_CUDA(cudaFuncSetAttribute(k_finish_bits<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_warp));
    }
    ZK_TRY(ctx->heavy_list.reserve((NB + 1) * 4));
    uint32_t *heavy_count = d_task_len + 1;       // cleared by k_pick_task_len
    k_combine_serial<F><<<(unsigned)((NB + 127) / 128), 128, 0, st>>>(partials, ctx->task_off.as<uint32_t>(), (uint32_t)NB, buckets,
                                                                      ctx->heavy_list.as<uint32_t>(), heavy_count);
    k_combine_warp<F><<<(unsigned)(2 * ctx->sm_count), 128, sm_warp, st>>>(partials, ctx->task_off.as<uint32_t>(), ctx->heavy_list.as<uint32_t>(), heavy_count, buckets);
    // 4. bucket reduction per domain
    XYZZ<F> *part = ctx->red_part.as<XYZZ<F>>(), *X = ctx->red_x.as<XYZZ<F>>(), *R = ctx->result.as<XYZZ<F>>();
    auto bit_reduce = [&](const XYZZ<F> *Bk, int N, int bits, size_t nd, XYZZ<F> *out) {     // out[dom] = sum_{d=1..N} d * Bk[dom][d-1]
        int slices = (N / 2 + RED_SLICE / 2 - 1) / (RED_SLICE / 2); if (slices < 1) slices = 1;
        size_t n_w = (size_t)slices * bits * nd, n_g = nd * (size_t)bits;
        k_bit_sums<F><<<(unsigned)((n_w * 32 + RED_T - 1) / RED_T), RED_T, sm_warp, st>>>(Bk, N, slices, bits, (int)nd, part);
        k_sum_points<F><<<(unsigned)((n_g * 32 + RED_T - 1) / RED_T), RED_T, sm_warp, st>>>(part, slices, (int)n_g, X);
        k_finish_bits<F><<<(unsigned)nd, FIN_WARPS * 32, 2 * FIN_WARPS * sizeof(XYZZ<F>), st>>>(X, bits, (int)nd, out);
    };
    XYZZ<F> *Rdom = tables ? R : R + 1;      // per-domain results; without tables they are the window sums the Horner pass folds into R[0]
    if ((n_dom >= 8 && c >= 7) || (tables && c > 16)) {
        // two-level row/column scheme, 2 additions per bucket (msm.cuh): many domains (batched proving) or wide windows
        const int s = (c - 1) / 2, nr = nbins >> s, nc = (1 << s) - 1;
        ZK_TRY(ctx->red_rows.reserve(2 * n_dom * (size_t)nr * pt));
        ZK_TRY(ctx->result.reserve((3 * n_dom + batch + 4) * pt));
        R = ctx->result.as<XYZZ<F>>();
        Rdom = tables ? R : R + 1;
        XYZZ<F> *rc = ctx->red_rows.as<XYZZ<F>>(), *Rrc = R + n_dom + 2;
        if (sm_warp > 48 * 1024) {
            ZK_CUDA(cudaFuncSetAttribute(k_rowcol_sums<F, RC_GL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_warp));
        }
        size_t n_items = n_dom * (size_t)(nr + nc);
        if (n_dom >= 8) {
            ZK_CUDA(cudaMemsetAsync(rc, 0, 2 * n_dom * (size_t)nr * pt, st));      // infinity padding of the column halves
            constexpr int per_warp = 32 / RC_GL;      // (domain, row / column) items per warp
            k_rowcol_sums<F, RC_GL><<<(unsigned)((((n_items + per_warp - 1) / per_warp) * 32 + RED_T - 1) / RED_T), RED_T, sm_warp, st>>>(buckets, nbins, s, (int)n_dom, rc);
        } else {
            const size_t n_slots = 2 * n_dom * (size_t)nr;
            const int longest = (1 << s) > nr + 1 ? (1 << s) : nr + 1;
            const int P1 = (longest + RC_L1 - 1) / RC_L1, P2 = (P1 + RC_L2 - 1) / RC_L2;
            ZK_TRY(ctx->red_tmp.reserve(n_slots * (size_t)(P1 + P2) * pt));
            XYZZ<F> *t1 = ctx->red_tmp.as<XYZZ<F>>(), *t2 = t1 + n_slots * P1;
            const int P1r = ((1 << s) + RC_L1 - 1) / RC_L1, P1c = (nr + 1 + RC_L1 - 1) / RC_L1;
            const size_t live = n_dom * ((size_t)nr * P1r + (size_t)nc * P1c);
            ZK_CUDA(cudaMemsetAsync(t1, 0, n_slots * (size_t)P1 * pt, st));
            k_rowcol_stage1<F><<<(unsigned)((live + RED_T - 1) / RED_T), RED_T, 0, st>>>(buckets, nbins, s, (int)n_dom, P1, t1);
            k_seg_sums<F><<<(unsigned)((n_slots * P2 + RED_T - 1) / RED_T), RED_T, 0, st>>>(t1, n_slots, P1, RC_L2, P2, t2);
            k_seg_sums<F><<<(unsigned)((n_slots + RED_T - 1) / RED_T), RED_T, 0, st>>>(t2, n_slots, P2, P2, 1, rc);
        }
        bit_reduce(rc, nr, c - s, 2 * n_dom, Rrc);      // rows: hi in [1, 2^(c-1-s)] (c-s bits); columns: lo in [1, 2^s - 1]
        k_join_rowcol<F><<<(unsigned)((n_dom * 32 + 127) / 128), 128, 0, st>>>(Rrc, s, (int)n_dom, Rdom);
    } else {
        bit_reduce(buckets, nbins, n_bits, n_dom, Rdom);
    }
    if (!tables) k_horner_windows<F><<<1, 32, 0, st>>>(Rdom, W, c, R);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

template <class F>
int encode_results_t(zk_ctx *ctx, size_t count, int compressed, uint8_t *d_out) {
    zkcodec::k_encode_xyzz<F><<<(unsigned)((count + 31) / 32), 32, 0, ctx->stream>>>(ctx->result.as<XYZZ<F>>(), (int)count, compressed, d_out);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

}  // namespace zkmsm
