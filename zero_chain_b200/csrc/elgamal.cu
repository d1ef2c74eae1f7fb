// Lifted-ElGamal balance decryption on the device (elgamal.cuh): zk_elgamal_decrypt_batch and its _device form.  The
// first call on a context builds the table of the 10^6 multiples of P_G and its index, which then stay resident in the
// context; every call after that runs one thread per ciphertext: up to four Point::reads with their subgroup tests, one
// 252-bit double-and-add, two inversions and a hash-table probe, all of it in registers.
//
// Like jubjub.cu, the translation unit holds only Fr / Fs arithmetic and is compiled with everything inlined (ZK_HOT).
#define ZK_HOT 1
#include "internal.h"
#include "elgamal.cuh"

using namespace zkeg;

constexpr int ET = 128;             // threads per block
constexpr int EG_BLOCKS_PER_SM = 8; // grid cap: larger batches loop over the grid

static __global__ void __launch_bounds__(ET) k_elgamal_table(uint32_t n, uint32_t *__restrict__ scratch, uint32_t *__restrict__ table) {
    eg_table_chunk(blockIdx.x * blockDim.x + threadIdx.x, n, scratch, table);
}

static __global__ void __launch_bounds__(ET) k_elgamal_index(uint32_t n, const uint32_t *__restrict__ table, uint32_t *__restrict__ index) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) eg_index_insert(index, EG_INDEX_MASK, table + 8 * (size_t)i, i);
}

static __global__ void __launch_bounds__(ET) k_elgamal_decrypt(size_t n, const uint8_t *__restrict__ dks, const uint8_t *__restrict__ cts,
                                                               const uint8_t *__restrict__ pending, const uint32_t *__restrict__ table,
                                                               const uint32_t *__restrict__ index, uint32_t *__restrict__ values,
                                                               uint8_t *__restrict__ status) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t v;
        status[i] = (uint8_t)elgamal_decrypt(dks + 32 * i, cts + 64 * i, pending ? pending + 64 * i : nullptr, table, index, EG_INDEX_MASK, v);
        values[i] = v;
    }
}

// The table (32 B per entry) and the index (4 B per slot), enqueued on the context's stream the first time they are needed
static int elgamal_tables(zk_ctx *ctx) {
    if (ctx->eg_ready) return ZK_OK;
    ZK_TRY(ctx->eg_table.reserve(32 * (size_t)EG_BOUND));
    ZK_TRY(ctx->eg_index.reserve(4 * ((size_t)EG_INDEX_MASK + 1)));
    uint32_t *table = ctx->eg_table.as<uint32_t>(), *index = ctx->eg_index.as<uint32_t>();
    void *scratch = nullptr;        // X, Y, Z of every entry, only while the chunks are normalised
    ZK_CUDA(cudaMallocAsync(&scratch, 96 * (size_t)EG_BOUND, ctx->stream));
    const uint32_t chunks = (EG_BOUND + EG_CHUNK - 1) / EG_CHUNK;
    k_elgamal_table<<<(chunks + ET - 1) / ET, ET, 0, ctx->stream>>>(EG_BOUND, static_cast<uint32_t *>(scratch), table);
    const cudaError_t launched = cudaGetLastError();
    ZK_CUDA(cudaFreeAsync(scratch, ctx->stream));
    ZK_CUDA(launched);
    ZK_CUDA(cudaMemsetAsync(index, 0xff, 4 * ((size_t)EG_INDEX_MASK + 1), ctx->stream));
    k_elgamal_index<<<(EG_BOUND + ET - 1) / ET, ET, 0, ctx->stream>>>(EG_BOUND, table, index);
    ZK_CUDA(cudaGetLastError());
    ctx->eg_ready = true;
    return ZK_OK;
}

static int launch_decrypt(zk_ctx *ctx, size_t n, const uint8_t *dks, const uint8_t *cts, const uint8_t *pending, uint32_t *values,
                          uint8_t *status) {
    ZK_TRY(elgamal_tables(ctx));
    const size_t cap = (size_t)(ctx->sm_count > 0 ? ctx->sm_count : 1) * EG_BLOCKS_PER_SM;
    const size_t blocks = (n + ET - 1) / ET < cap ? (n + ET - 1) / ET : cap;
    k_elgamal_decrypt<<<(unsigned)blocks, ET, 0, ctx->stream>>>(n, dks, cts, pending, ctx->eg_table.as<uint32_t>(),
                                                                ctx->eg_index.as<uint32_t>(), values, status);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

extern "C" int zk_elgamal_decrypt_batch_device(zk_ctx *ctx, size_t n, const uint8_t *d_dks, const uint8_t *d_cts, const uint8_t *d_pending,
                                               uint32_t *d_values, uint8_t *d_status) {
    if (!ctx || (n && (!d_dks || !d_cts || !d_values || !d_status))) {
        zk_set_error("zk_elgamal_decrypt_batch_device: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    return launch_decrypt(ctx, n, d_dks, d_cts, d_pending, d_values, d_status);
}

extern "C" int zk_elgamal_decrypt_batch(zk_ctx *ctx, size_t n, const uint8_t *dks, const uint8_t *cts, const uint8_t *pending,
                                        uint32_t *values, uint8_t *status) {
    if (!ctx || (n && (!dks || !cts || !values || !status))) {
        zk_set_error("zk_elgamal_decrypt_batch: NULL argument");
        return ZK_ERR_INVALID;
    }
    if (!n) return ZK_OK;
    ZK_TRY(zk_use_device(ctx));
    const uint8_t *d_dks, *d_cts, *d_pend;
    uint32_t *d_values;
    uint8_t *d_status;
    Stage io;
    io.in(dks, d_dks, 32 * n); io.in(cts, d_cts, 64 * n); io.in(pending, d_pend, 64 * n);
    io.out(values, d_values, n); io.out(status, d_status, n);
    ZK_TRY(io.up(ctx));
    ZK_TRY(launch_decrypt(ctx, n, d_dks, d_cts, d_pend, d_values, d_status));
    ZK_TRY(io.down(ctx));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}
