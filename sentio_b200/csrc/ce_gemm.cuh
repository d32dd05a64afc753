// ce_gemm.cuh -- interface of the wgmma GEMM used by the cross-encoder (ce_gemm.cu).
#pragma once
#include <cuda.h>

#include "common.cuh"

// CE_EPI_BIAS_RES16_F16: out16 = fp16(acc + bias + residual16) -- the all-fp16 residual stream of the reranker; `residual`
// then points at fp16 data (reinterpreted inside the kernels)
enum { CE_EPI_BIAS_F16 = 0, CE_EPI_BIAS_GELU_F16 = 1, CE_EPI_BIAS_RES_F32 = 2, CE_EPI_BIAS_RES16_F16 = 3 };

// 2-D tensor map over a row-major fp16 matrix [rows][cols] (cols contiguous), box 64 x 128, SWIZZLE_128B
int ce_make_tensor_map(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols);

// D[M,N] = A[M,K] * W[N,K]^T with one of the fused epilogues; M is padded to 128 by the caller's allocation.
// m_dev (may be NULL): device int holding the ACTUAL row count (<= M) -- the packed-token cross-encoder only knows its row
// count on the device; grids are sized for M and the kernels clamp their tile loops / stores to *m_dev.
int ce_gemm_launch(int epi, const CUtensorMap& map_a, const CUtensorMap& map_w, int M, int N, int K, const float* bias,
                   const float* residual, __half* out16, float* out32, cudaStream_t st, const int* m_dev = nullptr);
