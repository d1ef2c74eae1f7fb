// The few CUDA runtime names zero_chain_b200/csrc/internal.h uses, declared for a host-only build of it
// (tests/host_emul/emul_stage.cpp defines the functions over host memory).
#pragma once
#include <stddef.h>

enum cudaError_t { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
typedef struct CUstream_st *cudaStream_t;
typedef struct CUevent_st *cudaEvent_t;

cudaError_t cudaMalloc(void **p, size_t bytes);
cudaError_t cudaFree(void *p);
cudaError_t cudaMemcpyAsync(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, cudaStream_t stream);
const char *cudaGetErrorString(cudaError_t e);
