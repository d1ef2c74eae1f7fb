// Building confidential transfers on the device (tx_build.cuh): zk_keys_from_seed_batch, zk_g_epoch_batch,
// zk_confidential_fields_batch and zk_redjubjub_sign_batch, each with its _device form.  One thread per row, everything
// in registers; the fields call parks each row's seven points in a workspace of the context between its two passes and
// first builds the window table of the call's g_epoch with one thread per entry.  zk_anonymous_fields_batch decodes each key
// its rings name once, then runs a pass per row and a pass per (row, ring entry), so a row's 11 variable-base products
// spread over 11 threads.
//
// Like redjubjub.cu, the translation unit holds only Fr / Fs arithmetic and is compiled with everything inlined (ZK_HOT).
#define ZK_HOT 1
#include "internal.h"
#include "codec.cuh"
#include "tx_build.cuh"

using namespace zktb;

constexpr int TT = 128;             // threads per block
constexpr int TB_BLOCKS_PER_SM = 8; // grid cap: larger batches loop over the grid
constexpr int TB_SCRATCH_SLOTS = 28;

static __device__ __forceinline__ void load_le_words(const uint8_t *b, uint32_t *w, int n) {
#pragma unroll
    for (int i = 0; i < n; i++)     // byte loads: a device pointer passed in by the caller need not be word aligned
        w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
}
#define TB_ROWS(i, n) for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (size_t)gridDim.x * blockDim.x)

// seed i = seeds[off[i] - base .. off[i + 1] - base)
static __global__ void __launch_bounds__(TT) k_tb_keys(size_t n, const uint8_t *__restrict__ seeds, const uint64_t *__restrict__ off,
                                                       uint64_t base, uint8_t *__restrict__ sks, uint8_t *__restrict__ dks,
                                                       uint8_t *__restrict__ eks) {
    TB_ROWS(i, n) {
        const uint64_t o0 = off[i] - base, o1 = off[i + 1] - base;
        const Fs sk = spending_key(seeds + o0, o1 - o0);
        const Fs dk = decryption_key(sk);
        uint32_t ek[8];
        ext_encode(pg_mul(dk), ek);
        store_le_words(sks + 32 * i, sk.l, 8);
        store_le_words(dks + 32 * i, dk.l, 8);
        store_le_words(eks + 32 * i, ek, 8);
    }
}

// a row whose tag would reach 255 is left as 32 bytes of 0xff, which no Point::write produces
static __global__ void __launch_bounds__(TT) k_tb_g_epoch(size_t n, const uint32_t *__restrict__ epochs, uint8_t *__restrict__ out) {
    TB_ROWS(i, n) {
        uint32_t enc[8], tag;
        if (!g_epoch_hash(epochs[i], enc, tag))
            for (int k = 0; k < 8; k++) enc[k] = 0xffffffffu;
        store_le_words(out + 32 * i, enc, 8);
    }
}

// one thread per table entry; every thread reads g, and entry 0's thread reports a g that fails Point::read or
// as_prime_order through the context's decoding-error word (zk_check_err_flag turns DEC_NOT_ON_CURVE into ZK_ERR_DECODE)
static __global__ void __launch_bounds__(TT) k_tb_epoch_table(const uint8_t *__restrict__ g_enc, uint32_t *__restrict__ table, int *err) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= TB_WINDOWS * TB_DIGITS) return;
    uint32_t w[8];
    load_le_words(g_enc, w, 8);
    Ext g;
    if (read_prime_order(w, g) != JJ_OK) {
        if (e == 0) atomicExch(err, zkcodec::DEC_NOT_ON_CURVE);
        g = ext_identity();
    }
    tb_epoch_entry(g, e, table + TB_ENTRY_WORDS * e);
}

static __global__ void __launch_bounds__(TT) k_tb_fields(size_t n, const uint8_t *__restrict__ sks, const uint8_t *__restrict__ eks,
                                                         const uint32_t *__restrict__ amounts, const uint32_t *__restrict__ fees,
                                                         const uint8_t *__restrict__ rs, const uint8_t *__restrict__ alphas,
                                                         const uint8_t *__restrict__ g_enc, const uint32_t *__restrict__ table,
                                                         uint32_t *__restrict__ scratch, uint8_t *__restrict__ fields,
                                                         uint8_t *__restrict__ rsks, uint8_t *__restrict__ dks, uint8_t *__restrict__ status,
                                                         int *not_canonical) {
    TB_ROWS(i, n) {
        uint32_t sk[8], ek[8], r[8], al[8];
        load_le_words(sks + 32 * i, sk, 8); load_le_words(eks + 32 * i, ek, 8);
        load_le_words(rs + 32 * i, r, 8); load_le_words(alphas + 32 * i, al, 8);
        if (!Fs::canonical_lt_mod(fs_words(sk)) || !Fs::canonical_lt_mod(fs_words(r)) || !Fs::canonical_lt_mod(fs_words(al))) {
            atomicExch(not_canonical, 1);
            continue;
        }
        status[i] = (uint8_t)confidential_fields(sk, ek, amounts[i], fees[i], r, al, g_enc, table, scratch + i, n, fields + 32 * TB_N_FIELDS * i,
                                                 rsks + 32 * i, dks + 32 * i);
    }
}

static __global__ void __launch_bounds__(TT) k_tb_sign(size_t n, const uint8_t *__restrict__ sks, const uint8_t *__restrict__ ts,
                                                       const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off, uint64_t base,
                                                       uint8_t *__restrict__ sigs, int *not_canonical) {
    TB_ROWS(i, n) {
        uint32_t sk[8], tw[20], sig[16];
        load_le_words(sks + 32 * i, sk, 8);
        load_le_words(ts + 80 * i, tw, 20);
        if (!Fs::canonical_lt_mod(fs_words(sk))) {
            atomicExch(not_canonical, 1);
            continue;
        }
        uint64_t t[10];
#pragma unroll
        for (int k = 0; k < 10; k++) t[k] = (uint64_t)tw[2 * k] | ((uint64_t)tw[2 * k + 1] << 32);
        const uint64_t o0 = off[i] - base, o1 = off[i + 1] - base;
        redjubjub_sign(fs_words(sk), t, msgs + o0, o1 - o0, sig);
        store_le_words(sigs + 64 * i, sig, 16);
    }
}

// ---- zk_anonymous_fields_batch: the key table, then the row pass, then the left pass -------------------------------------
// one thread per ring index: flags each key an in-range index names (named[] zeroed before)
static __global__ void __launch_bounds__(TT) k_tb_anon_named(size_t m, const uint32_t *__restrict__ rings, size_t n_keys,
                                                             uint8_t *__restrict__ named) {
    TB_ROWS(k, m) {
        const uint32_t idx = rings[k];
        if (idx < n_keys) named[idx] = 1;
    }
}

// one thread per key: a named key is read once, whatever number of rows name it; the others are left alone
static __global__ void __launch_bounds__(TT) k_tb_anon_keys(size_t n_keys, const uint8_t *__restrict__ keys, const uint8_t *__restrict__ named,
                                                            uint32_t *__restrict__ niels, uint8_t *__restrict__ key_status) {
    TB_ROWS(k, n_keys) {
        if (!named[k]) continue;
        uint32_t w[8];
        load_le_words(keys + 32 * k, w, 8);
        key_status[k] = (uint8_t)anon_key_entry(w, niels + TB_ENTRY_WORDS * k);
    }
}

static __device__ __forceinline__ bool anon_canonical(size_t i, const uint8_t *sks, const uint8_t *rs, const uint8_t *alphas, uint32_t *sk,
                                                      uint32_t *r, uint32_t *al) {
    load_le_words(sks + 32 * i, sk, 8); load_le_words(rs + 32 * i, r, 8); load_le_words(alphas + 32 * i, al, 8);
    return Fs::canonical_lt_mod(fs_words(sk)) && Fs::canonical_lt_mod(fs_words(r)) && Fs::canonical_lt_mod(fs_words(al));
}

static __global__ void __launch_bounds__(TT) k_tb_anon_rows(size_t n, const uint8_t *__restrict__ sks, const uint32_t *__restrict__ rings,
                                                            const uint8_t *__restrict__ positions, const uint32_t *__restrict__ amounts,
                                                            const uint8_t *__restrict__ rs, const uint8_t *__restrict__ alphas, size_t n_keys,
                                                            const uint8_t *__restrict__ key_status, const uint32_t *__restrict__ table,
                                                            uint32_t *__restrict__ scratch, uint8_t *__restrict__ fields,
                                                            uint8_t *__restrict__ rsks, uint8_t *__restrict__ dks, uint8_t *__restrict__ status,
                                                            int *not_canonical) {
    TB_ROWS(i, n) {
        uint32_t sk[8], r[8], al[8];
        if (!anon_canonical(i, sks, rs, alphas, sk, r, al)) {
            atomicExch(not_canonical, 1);
            continue;
        }
        const int s = positions[2 * i], t = positions[2 * i + 1];
        const int st = anon_status(s, t, rings + (size_t)TB_RING_IN * i, n_keys, key_status);
        anonymous_row(st, s, sk, amounts[i], r, al, table, scratch + i, n, fields + 32 * TB_N_ANON_FIELDS * i, rsks + 32 * i, dks + 32 * i);
        status[i] = (uint8_t)st;
    }
}

// thread TB_RING_IN i + j: ring entry j of row i, so a row's entries run side by side; rows the row pass refused (status)
// or skipped (a scalar >= r_J) are left as it left them
static __global__ void __launch_bounds__(TT) k_tb_anon_lefts(size_t n, const uint8_t *__restrict__ keys, const uint32_t *__restrict__ rings,
                                                             const uint8_t *__restrict__ positions, const uint32_t *__restrict__ amounts,
                                                             const uint8_t *__restrict__ sks, const uint8_t *__restrict__ rs,
                                                             const uint8_t *__restrict__ alphas, const uint32_t *__restrict__ niels,
                                                             const uint8_t *__restrict__ status, uint8_t *__restrict__ fields) {
    TB_ROWS(k, TB_RING_IN * n) {
        const size_t i = k / TB_RING_IN;
        const int j = (int)(k - TB_RING_IN * i);
        uint32_t sk[8], r[8], al[8];
        if (!anon_canonical(i, sks, rs, alphas, sk, r, al) || status[i] != JJ_OK) continue;
        const size_t idx = rings[k];
        anonymous_left(load_niels(niels + TB_ENTRY_WORDS * idx), keys + 32 * idx, j, anon_position(positions[2 * i], positions[2 * i + 1], j),
                       amounts[i], r, fields + 32 * TB_N_ANON_FIELDS * i);
    }
}

static unsigned grid(const zk_ctx *ctx, size_t n) {
    const size_t cap = (size_t)(ctx->sm_count > 0 ? ctx->sm_count : 1) * TB_BLOCKS_PER_SM;
    return (unsigned)((n + TT - 1) / TT < cap ? (n + TT - 1) / TT : cap);
}

// ---- host-side checks -------------------------------------------------------------------------------------------------
static bool fs_canonical(const uint8_t *b) {   // little-endian 32 bytes < r_J
    static const uint32_t r_j[8] = {0xd6f72cb7u, 0xd0970e5eu, 0xccc81082u, 0xa6682093u, 0x01343b00u, 0x06673b01u, 0x6533afa9u, 0x0e7db4eau};
    for (int i = 31; i >= 0; i--) {
        const uint8_t m = (uint8_t)(r_j[i / 4] >> (8 * (i % 4)));
        if (b[i] != m) return b[i] < m;
    }
    return false;
}
static int check_scalars(const char *fn, const char *what, size_t n, const uint8_t *s) {
    for (size_t i = 0; i < n; i++)
        if (!fs_canonical(s + 32 * i)) {
            zk_set_error("%s: %s[%zu] >= r_J", fn, what, i);
            return ZK_ERR_NOT_CANONICAL;
        }
    return ZK_OK;
}
static int check_offsets(const char *fn, size_t n, const uint64_t *off) {
    for (size_t i = 0; i < n; i++)
        if (off[i + 1] < off[i]) {
            zk_set_error("%s: off[%zu] = %llu > off[%zu] = %llu", fn, i, (unsigned long long)off[i], i + 1, (unsigned long long)off[i + 1]);
            return ZK_ERR_INVALID;
        }
    return ZK_OK;
}

// ---- zk_keys_from_seed_batch ----------------------------------------------------------------------------------------------
extern "C" int zk_keys_from_seed_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_seeds, const uint64_t *d_seed_off, uint8_t *d_sks,
                                              uint8_t *d_dks, uint8_t *d_eks) {
    if (!ctx || (n && (!d_seeds || !d_seed_off || !d_sks || !d_dks || !d_eks))) {
        zk_set_error("zk_keys_from_seed_batch_device: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    k_tb_keys<<<grid(ctx, n), TT, 0, ctx->stream>>>(n, d_seeds, d_seed_off, 0, d_sks, d_dks, d_eks);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_keys_from_seed_batch(zk_ctx *ctx, size_t n, const uint8_t *seeds, const uint64_t *seed_off, uint8_t *sks, uint8_t *dks,
                                       uint8_t *eks) {
    if (!ctx || (n && (!seeds || !seed_off || !sks || !dks || !eks))) {
        zk_set_error("zk_keys_from_seed_batch: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(check_offsets("zk_keys_from_seed_batch", n, seed_off));
    ZK_TRY(zk_use_device(ctx));
    const uint64_t base = seed_off[0];
    const uint8_t *d_seeds;
    const uint64_t *d_off;
    uint8_t *d_sks, *d_dks, *d_eks;
    Stage io;
    io.in(seed_off, d_off, n + 1); io.in(seeds + base, d_seeds, seed_off[n] - base);
    io.out(sks, d_sks, 32 * n); io.out(dks, d_dks, 32 * n); io.out(eks, d_eks, 32 * n);
    ZK_TRY(io.up(ctx));
    k_tb_keys<<<grid(ctx, n), TT, 0, ctx->stream>>>(n, d_seeds, d_off, base, d_sks, d_dks, d_eks);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

// ---- zk_g_epoch_batch -----------------------------------------------------------------------------------------------------
extern "C" int zk_g_epoch_batch_device(zk_ctx *ctx, size_t n, const uint32_t *d_epochs, uint8_t *d_g_epochs) {
    if (!ctx || (n && (!d_epochs || !d_g_epochs))) {
        zk_set_error("zk_g_epoch_batch_device: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    k_tb_g_epoch<<<grid(ctx, n), TT, 0, ctx->stream>>>(n, d_epochs, d_g_epochs);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_g_epoch_batch(zk_ctx *ctx, size_t n, const uint32_t *epochs, uint8_t *g_epochs) {
    if (!ctx || (n && (!epochs || !g_epochs))) {
        zk_set_error("zk_g_epoch_batch: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint32_t *d_epochs;
    uint8_t *d_out;
    Stage io;
    io.in(epochs, d_epochs, n); io.out(g_epochs, d_out, 32 * n);
    ZK_TRY(io.up(ctx));
    k_tb_g_epoch<<<grid(ctx, n), TT, 0, ctx->stream>>>(n, d_epochs, d_out);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < n; i++) {
        bool all = true;
        for (int k = 0; k < 32; k++) all = all && g_epochs[32 * i + k] == 0xff;
        if (all) {
            zk_set_error("zk_g_epoch_batch: GEpoch::group_hash(%u) finds no point below tag byte 255", epochs[i]);
            return ZK_ERR_DECODE;
        }
    }
    return ZK_OK;
}

// ---- zk_confidential_fields_batch -----------------------------------------------------------------------------------------
static int launch_fields(zk_ctx *ctx, size_t n, const uint8_t *sks, const uint8_t *eks, const uint32_t *amounts, const uint32_t *fees,
                         const uint8_t *rs, const uint8_t *alphas, const uint8_t *g_epoch, uint8_t *fields, uint8_t *rsks, uint8_t *dks,
                         uint8_t *status) {
    Carve sizing;
    sizing.take<uint32_t>(TB_TABLE_WORDS); sizing.take<uint32_t>(8 * TB_SCRATCH_SLOTS * n);
    ZK_TRY(ctx->tb.reserve(sizing.off));
    Carve c{ctx->tb.as<uint8_t>(), 0};
    uint32_t *table = c.take<uint32_t>(TB_TABLE_WORDS), *scratch = c.take<uint32_t>(8 * TB_SCRATCH_SLOTS * n);
    k_tb_epoch_table<<<(TB_WINDOWS * TB_DIGITS + TT - 1) / TT, TT, 0, ctx->stream>>>(g_epoch, table, ctx->d_err + 1);
    ZK_CUDA(cudaGetLastError());
    k_tb_fields<<<grid(ctx, n), TT, 0, ctx->stream>>>(n, sks, eks, amounts, fees, rs, alphas, g_epoch, table, scratch, fields, rsks, dks, status,
                                                      ctx->d_err);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_confidential_fields_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_sks, const uint8_t *d_eks_recipient,
                                                   const uint32_t *d_amounts, const uint32_t *d_fees, const uint8_t *d_rs,
                                                   const uint8_t *d_alphas, const uint8_t *d_g_epoch, uint8_t *d_fields, uint8_t *d_rsks,
                                                   uint8_t *d_dks, uint8_t *d_status) {
    if (!ctx || (n && (!d_sks || !d_eks_recipient || !d_amounts || !d_fees || !d_rs || !d_alphas || !d_g_epoch || !d_fields || !d_rsks ||
                       !d_dks || !d_status))) {
        zk_set_error("zk_confidential_fields_batch_device: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return launch_fields(ctx, n, d_sks, d_eks_recipient, d_amounts, d_fees, d_rs, d_alphas, d_g_epoch, d_fields, d_rsks, d_dks, d_status);
}

extern "C" int zk_confidential_fields_batch(zk_ctx *ctx, size_t n, const uint8_t *sks, const uint8_t *eks_recipient, const uint32_t *amounts,
                                            const uint32_t *fees, const uint8_t *rs, const uint8_t *alphas, const uint8_t *g_epoch,
                                            uint8_t *fields, uint8_t *rsks, uint8_t *dks, uint8_t *status) {
    static const char *fn = "zk_confidential_fields_batch";
    if (!ctx || (n && (!sks || !eks_recipient || !amounts || !fees || !rs || !alphas || !g_epoch || !fields || !rsks || !dks || !status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(check_scalars(fn, "sks", n, sks));
    ZK_TRY(check_scalars(fn, "rs", n, rs));
    ZK_TRY(check_scalars(fn, "alphas", n, alphas));
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d_sks, *d_eks, *d_rs, *d_al, *d_g;
    const uint32_t *d_am, *d_fee;
    uint8_t *d_fields, *d_rsks, *d_dks, *d_st;
    Stage io;
    io.in(sks, d_sks, 32 * n); io.in(eks_recipient, d_eks, 32 * n); io.in(amounts, d_am, n); io.in(fees, d_fee, n);
    io.in(rs, d_rs, 32 * n); io.in(alphas, d_al, 32 * n); io.in(g_epoch, d_g, 32);
    io.out(fields, d_fields, 32 * TB_N_FIELDS * n); io.out(rsks, d_rsks, 32 * n); io.out(dks, d_dks, 32 * n); io.out(status, d_st, n);
    ZK_TRY(io.up(ctx));
    ZK_TRY(launch_fields(ctx, n, d_sks, d_eks, d_am, d_fee, d_rs, d_al, d_g, d_fields, d_rsks, d_dks, d_st));
    ZK_TRY(io.down(ctx));
    const int rc = zk_check_err_flag(ctx);   // synchronises the stream
    if (rc == ZK_ERR_DECODE) zk_set_error("%s: g_epoch fails Point::read or is not of prime order", fn);
    return rc;
}

// ---- zk_anonymous_fields_batch --------------------------------------------------------------------------------------------
constexpr size_t TB_ANON_MAX_ROWS = (size_t)1 << 22, TB_ANON_MAX_KEYS = (size_t)1 << 24;

static int check_anon_sizes(const char *fn, size_t n_keys, size_t n) {
    if (n > TB_ANON_MAX_ROWS || n_keys > TB_ANON_MAX_KEYS) {
        zk_set_error("%s: n = %zu, n_keys = %zu; at most 2^22 rows and 2^24 keys", fn, n, n_keys);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

static int launch_anon(zk_ctx *ctx, size_t n_keys, const uint8_t *keys, size_t n, const uint8_t *sks, const uint32_t *rings,
                       const uint8_t *positions, const uint32_t *amounts, const uint8_t *rs, const uint8_t *alphas, const uint8_t *g_epoch,
                       uint8_t *fields, uint8_t *rsks, uint8_t *dks, uint8_t *status) {
    Carve sizing;
    sizing.take<uint32_t>(TB_TABLE_WORDS); sizing.take<uint32_t>(8 * TB_ANON_SCRATCH_SLOTS * n);
    sizing.take<uint32_t>(TB_ENTRY_WORDS * n_keys); sizing.take<uint8_t>(n_keys); sizing.take<uint8_t>(n_keys);
    ZK_TRY(ctx->tb.reserve(sizing.off));
    Carve c{ctx->tb.as<uint8_t>(), 0};
    uint32_t *table = c.take<uint32_t>(TB_TABLE_WORDS), *scratch = c.take<uint32_t>(8 * TB_ANON_SCRATCH_SLOTS * n);
    uint32_t *niels = c.take<uint32_t>(TB_ENTRY_WORDS * n_keys);
    uint8_t *named = c.take<uint8_t>(n_keys), *key_status = c.take<uint8_t>(n_keys);
    k_tb_epoch_table<<<(TB_WINDOWS * TB_DIGITS + TT - 1) / TT, TT, 0, ctx->stream>>>(g_epoch, table, ctx->d_err + 1);
    ZK_CUDA(cudaGetLastError());
    if (n_keys) {
        ZK_CUDA(cudaMemsetAsync(named, 0, n_keys, ctx->stream));
        k_tb_anon_named<<<grid(ctx, TB_RING_IN * n), TT, 0, ctx->stream>>>(TB_RING_IN * n, rings, n_keys, named);
        ZK_CUDA(cudaGetLastError());
        k_tb_anon_keys<<<grid(ctx, n_keys), TT, 0, ctx->stream>>>(n_keys, keys, named, niels, key_status);
        ZK_CUDA(cudaGetLastError());
    }
    k_tb_anon_rows<<<grid(ctx, n), TT, 0, ctx->stream>>>(n, sks, rings, positions, amounts, rs, alphas, n_keys, key_status, table, scratch,
                                                         fields, rsks, dks, status, ctx->d_err);
    ZK_CUDA(cudaGetLastError());
    k_tb_anon_lefts<<<grid(ctx, TB_RING_IN * n), TT, 0, ctx->stream>>>(n, keys, rings, positions, amounts, sks, rs, alphas, niels, status,
                                                                       fields);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_anonymous_fields_batch_device(zk_ctx *ctx, size_t n_keys, const uint8_t *d_keys, size_t n, const uint8_t *d_sks,
                                                const uint32_t *d_rings, const uint8_t *d_positions, const uint32_t *d_amounts,
                                                const uint8_t *d_rs, const uint8_t *d_alphas, const uint8_t *d_g_epoch, uint8_t *d_fields,
                                                uint8_t *d_rsks, uint8_t *d_dks, uint8_t *d_status) {
    static const char *fn = "zk_anonymous_fields_batch_device";
    if (!ctx || (n_keys && !d_keys) || (n && (!d_sks || !d_rings || !d_positions || !d_amounts || !d_rs || !d_alphas || !d_g_epoch ||
                                              !d_fields || !d_rsks || !d_dks || !d_status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    ZK_TRY(check_anon_sizes(fn, n_keys, n));
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return launch_anon(ctx, n_keys, d_keys, n, d_sks, d_rings, d_positions, d_amounts, d_rs, d_alphas, d_g_epoch, d_fields, d_rsks, d_dks,
                       d_status);
}

extern "C" int zk_anonymous_fields_batch(zk_ctx *ctx, size_t n_keys, const uint8_t *keys, size_t n, const uint8_t *sks, const uint32_t *rings,
                                         const uint8_t *positions, const uint32_t *amounts, const uint8_t *rs, const uint8_t *alphas,
                                         const uint8_t *g_epoch, uint8_t *fields, uint8_t *rsks, uint8_t *dks, uint8_t *status) {
    static const char *fn = "zk_anonymous_fields_batch";
    if (!ctx || (n_keys && !keys) || (n && (!sks || !rings || !positions || !amounts || !rs || !alphas || !g_epoch || !fields || !rsks ||
                                            !dks || !status))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    ZK_TRY(check_anon_sizes(fn, n_keys, n));
    if (!n) return ZK_OK;
    ZK_TRY(check_scalars(fn, "sks", n, sks));
    ZK_TRY(check_scalars(fn, "rs", n, rs));
    ZK_TRY(check_scalars(fn, "alphas", n, alphas));
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d_keys, *d_sks, *d_pos, *d_rs, *d_al, *d_g;
    const uint32_t *d_rings, *d_am;
    uint8_t *d_fields, *d_rsks, *d_dks, *d_st;
    Stage io;
    io.in(keys, d_keys, 32 * n_keys); io.in(sks, d_sks, 32 * n); io.in(rings, d_rings, TB_RING_IN * n); io.in(positions, d_pos, 2 * n);
    io.in(amounts, d_am, n); io.in(rs, d_rs, 32 * n); io.in(alphas, d_al, 32 * n); io.in(g_epoch, d_g, 32);
    io.out(fields, d_fields, 32 * TB_N_ANON_FIELDS * n); io.out(rsks, d_rsks, 32 * n); io.out(dks, d_dks, 32 * n); io.out(status, d_st, n);
    ZK_TRY(io.up(ctx));
    ZK_TRY(launch_anon(ctx, n_keys, d_keys, n, d_sks, d_rings, d_pos, d_am, d_rs, d_al, d_g, d_fields, d_rsks, d_dks, d_st));
    ZK_TRY(io.down(ctx));
    const int rc = zk_check_err_flag(ctx);   // synchronises the stream
    if (rc == ZK_ERR_DECODE) zk_set_error("%s: g_epoch fails Point::read or is not of prime order", fn);
    return rc;
}

// ---- zk_redjubjub_sign_batch ----------------------------------------------------------------------------------------------
extern "C" int zk_redjubjub_sign_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_sks, const uint8_t *d_ts, const uint8_t *d_msgs,
                                              const uint64_t *d_msg_off, uint8_t *d_sigs) {
    if (!ctx || (n && (!d_sks || !d_ts || !d_msgs || !d_msg_off || !d_sigs))) {
        zk_set_error("zk_redjubjub_sign_batch_device: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    k_tb_sign<<<grid(ctx, n), TT, 0, ctx->stream>>>(n, d_sks, d_ts, d_msgs, d_msg_off, 0, d_sigs, ctx->d_err);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_redjubjub_sign_batch(zk_ctx *ctx, size_t n, const uint8_t *sks, const uint8_t *ts, const uint8_t *msgs, const uint64_t *msg_off,
                                       uint8_t *sigs) {
    static const char *fn = "zk_redjubjub_sign_batch";
    if (!ctx || (n && (!sks || !ts || !msgs || !msg_off || !sigs))) {
        zk_set_error("%s: NULL argument", fn);
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(check_offsets(fn, n, msg_off));
    ZK_TRY(check_scalars(fn, "sks", n, sks));
    ZK_TRY(zk_use_device(ctx));
    const uint64_t base = msg_off[0];
    const uint8_t *d_sks, *d_ts, *d_msgs;
    const uint64_t *d_off;
    uint8_t *d_sigs;
    Stage io;
    io.in(msg_off, d_off, n + 1); io.in(sks, d_sks, 32 * n); io.in(ts, d_ts, 80 * n); io.in(msgs + base, d_msgs, msg_off[n] - base);
    io.out(sigs, d_sigs, 64 * n);
    ZK_TRY(io.up(ctx));
    k_tb_sign<<<grid(ctx, n), TT, 0, ctx->stream>>>(n, d_sks, d_ts, d_msgs, d_off, base, d_sigs, ctx->d_err);
    ZK_CUDA(cudaGetLastError());
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}
