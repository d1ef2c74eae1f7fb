// CPU harness of the host forms' staging (Stage in zero_chain_b200/csrc/internal.h), built with g++ against the CUDA stub
// in cuda_stub/: cudaMalloc / cudaFree work on host memory and are counted, cudaMemcpyAsync copies at once and records
// each copy.  tests/test_host_stage.py registers arrays of every direction, size and element type through emu_up, writes
// the "run"'s results into the device copies, and checks emu_down's copies.
#include "internal.h"

#include <memory>
#include <stdlib.h>

struct Copy { int kind; const void *dst, *src; size_t bytes; };
static std::vector<Copy> g_log;
static size_t g_mallocs = 0;
static zk_ctx g_ctx;
static std::unique_ptr<Stage> g_stage;
static std::vector<uint8_t *> g_d8;
static std::vector<uint32_t *> g_d32;
static std::vector<const uint64_t *> g_d64;    // a const device pointer, as the host forms use for their inputs

cudaError_t cudaMalloc(void **p, size_t bytes) {
    *p = aligned_alloc(256, (bytes + 255) & ~(size_t)255);
    g_mallocs++;
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, cudaStream_t) {
    g_log.push_back({kind, dst, src, bytes});
    memcpy(dst, src, bytes);
    return cudaSuccess;
}
const char *cudaGetErrorString(cudaError_t) { return "stub error"; }
void zk_set_error(const char *, ...) {}

extern "C" {
// dir[i]: 1 in, 2 out, 3 in-out; elem[i]: 1, 4 or 8 bytes (8: inputs only); host[i] may be NULL; width[i] > 0: an output
// that comes down for *rows rows of width[i] elements.  dev[i]: the device pointer up() filled in (0: NULL); every device
// pointer starts non-NULL.
int emu_up(size_t n, const int *dir, const size_t *elem, const size_t *count, void *const *host, const size_t *width, const size_t *rows,
           uint64_t *dev) {
    g_stage.reset(new Stage);
    g_d8.assign(n, reinterpret_cast<uint8_t *>(1));
    g_d32.assign(n, reinterpret_cast<uint32_t *>(1));
    g_d64.assign(n, reinterpret_cast<const uint64_t *>(1));
    Stage &io = *g_stage;
    for (size_t i = 0; i < n; i++) {
        const size_t *r = width[i] ? rows : nullptr;
        const size_t w = width[i] ? width[i] : 1;
        if (elem[i] == 1) {
            uint8_t *h = static_cast<uint8_t *>(host[i]);
            if (dir[i] == 1) io.in(h, g_d8[i], count[i]); else if (dir[i] == 2) io.out(h, g_d8[i], count[i], r, w); else io.inout(h, g_d8[i], count[i]);
        } else if (elem[i] == 4) {
            uint32_t *h = static_cast<uint32_t *>(host[i]);
            if (dir[i] == 1) io.in(h, g_d32[i], count[i]); else if (dir[i] == 2) io.out(h, g_d32[i], count[i], r, w); else io.inout(h, g_d32[i], count[i]);
        } else {
            const uint64_t *h = static_cast<const uint64_t *>(host[i]);
            if (dir[i] != 1) return -100;
            io.in(h, g_d64[i], count[i]);
        }
    }
    const int rc = io.up(&g_ctx);
    for (size_t i = 0; i < n; i++)
        dev[i] = (uint64_t)(elem[i] == 1 ? (uintptr_t)g_d8[i] : elem[i] == 4 ? (uintptr_t)g_d32[i] : (uintptr_t)g_d64[i]);
    return rc;
}
int emu_down() { return g_stage->down(&g_ctx); }

// the copies since the last call: kind, dst, src, bytes
size_t emu_copies(int *kind, uint64_t *dst, uint64_t *src, uint64_t *bytes, size_t cap) {
    const size_t n = g_log.size();
    for (size_t i = 0; i < n && i < cap; i++) {
        kind[i] = g_log[i].kind; dst[i] = (uintptr_t)g_log[i].dst; src[i] = (uintptr_t)g_log[i].src; bytes[i] = g_log[i].bytes;
    }
    g_log.clear();
    return n;
}
size_t emu_mallocs() { return g_mallocs; }
uint64_t emu_io_base() { return (uintptr_t)g_ctx.io.p; }
size_t emu_io_cap() { return g_ctx.io.cap; }
}
