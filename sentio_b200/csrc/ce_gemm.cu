// ce_gemm.cu -- wgmma / TMA GEMM for the cross-encoder (K5):  D[M,N] = A[M,K] * W[N,K]^T  (+ epilogue), sm_90a
//
// A (activations) and W (nn.Linear weights) are both K-major fp16, accumulation is fp32 in registers.
// One 128 x 128 output tile per CTA, K consumed in 64-element (128-byte, SWIZZLE_128B) chunks through a 3-stage
// TMA -> mbarrier -> wgmma ring.  Warp roles: warps 0..7 = two consumer warpgroups (warpgroup g owns output rows
// [64 g, 64 g + 64) of the tile: m64n128k16 MMAs, then the epilogue straight from the accumulator registers),
// warp 8 = TMA producer (one elected lane).  Two CTAs are resident per SM (97 KB shared memory and 288 threads each),
// so one tile's epilogue overlaps another's mainloop.
//
// Epilogues:  BIAS_F16        out16 = acc + bias                      (QKV projection)
//             BIAS_GELU_F16   out16 = gelu_erf(acc + bias)            (FFN up-projection)
//             BIAS_RES_F32    out32 = acc + bias + residual32         (attention output / FFN down-projection, pre-LN)
//             BIAS_RES16_F16  out16 = fp16(acc + bias + residual16)   (the same two GEMMs on the fp16 residual stream:
//                             half the epilogue bytes; the pre-LN sum is rounded to fp16 once)
//
// Bound: tensor pipe (2*M*N*K flops); see DESIGN.md for the per-pair flop count.
#include <cuda.h>
#include <stdlib.h>

#include <algorithm>

#include "ce_gemm.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int kStages = 3;
constexpr int kConsumerThreads = 256;                  // two warpgroups
constexpr int kGemmThreads = kConsumerThreads + 32;    // + the TMA producer warp
constexpr uint32_t kTileABytes = BM * BK * 2, kTileBBytes = BN * BK * 2;
constexpr uint32_t kStageBytes = kTileABytes + kTileBBytes;
constexpr size_t kGemmSmem = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}

// erf-GELU (the HuggingFace "gelu") = 0.5 x (1 + erf(x / sqrt 2)), evaluated on a PAIR of outputs in packed half precision
// with ONE transcendental:  erf(x / sqrt 2) ~ tanh(x (c0 + c1 x^2 + c2 x^4)),  c fitted by least squares on the GELU itself
// over |x| <= 5.5 (scripts/fit_gelu.py): max |error| 3.0e-5 in exact arithmetic -- 16 x below the stock "tanh GELU"
// (4.7e-4) and below half an fp16 ulp of the result wherever |gelu| > 0.06.  8 packed instructions per pair
// (HMUL2 HMNMX2 2 x HFMA2 HMUL2 MUFU.TANH HMUL2 HFMA2); x^2 is clamped at 36 where tanh has saturated in fp16.
// Error study (scripts/fit_gelu.py, every operation rounded to fp16, tanh with the
// 2^-11 relative error of tanh.approx): rms |error| 2.0e-4 on N(0,1) inputs vs 2.6e-4 for the A-S form and 1.3e-4 for the
// exact function rounded to fp16 -- the storage rounding dominates either way (tolerance of the path: 1e-3 on the score).
__device__ __forceinline__ __half2 gelu_erf_h2(__half2 x) {
  const __half2 x2 = __hmin2(__hmul2(x, x), __float2half2_rn(36.0f));
  __half2 q = __hfma2(__float2half2_rn(-0.00035873236644f), x2, __float2half2_rn(0.0370503451315f));
  q = __hfma2(q, x2, __float2half2_rn(0.79745847075f));
  const __half2 u = __hmul2(x, q);
  uint32_t tb;
  const uint32_t ub = *reinterpret_cast<const uint32_t*>(&u);
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(tb) : "r"(ub));
  const __half2 th = *reinterpret_cast<const __half2*>(&tb);
  const __half2 hx = __hmul2(__float2half2_rn(0.5f), x);
  return __hfma2(hx, th, hx);
}
// bias-added fp32 pair -> fp16 pair, through the activation of the epilogue
template <int EPI>
__device__ __forceinline__ __half2 act_pack(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return EPI == CE_EPI_BIAS_GELU_F16 ? gelu_erf_h2(h) : h;
}

template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 2)
ce_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, int M_cap, int N, int K,
               const float* __restrict__ bias, const float* __restrict__ residual, __half* __restrict__ out16,
               float* __restrict__ out32, const int* __restrict__ m_dev) {
  const int M = m_dev ? min(M_cap, __ldg(m_dev)) : M_cap;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  if (m0 >= M) return;  // the device-side row count left this tile empty (uniform over the CTA)
  extern __shared__ uint8_t gsm_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t raw = smem_u32(gsm_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gsm = gsm_raw + (base - raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(gsm + kStages * kStageBytes);
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + kStages);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_k = K / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, kConsumerThreads / 32);   // one arrival per consumer warp
    }
    mbar_fence_init();
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
  }
  __syncthreads();

  if (warp == kConsumerThreads / 32) {
    // ---------------------------------------------------------------- TMA producer
    if (lane == 0) {
      for (int kb = 0; kb < num_k; ++kb) {
        const int s = kb % kStages;
        const uint32_t use = (uint32_t)(kb / kStages);
        if (kb >= kStages) mbar_wait(bar_empty + 8 * s, (use & 1u) ^ 1u);
        const uint32_t sa = base + (uint32_t)s * kStageBytes, sb = sa + kTileABytes;
        mbar_expect_tx(bar_full + 8 * s, kStageBytes);
        tma_load_2d(sa, &map_a, kb * BK, m0, bar_full + 8 * s);
        tma_load_2d(sb, &map_w, kb * BK, n0, bar_full + 8 * s);
      }
    }
    return;
  }
  // ---------------------------------------------------------------- consumer warpgroups: MMA, then the epilogue
  const int wg = warp >> 2;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < num_k; ++kb) {
    const int s = kb % kStages;
    mbar_wait(bar_full + 8 * s, (uint32_t)(kb / kStages) & 1u);
    const uint32_t sa = base + (uint32_t)s * kStageBytes + (uint32_t)wg * (kTileABytes / 2), sb = base + (uint32_t)s * kStageBytes + kTileABytes;
    const uint64_t da = wgmma_desc_sw128(sa), db = wgmma_desc_sw128(sb);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) Wgmma<BN>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) ? 1u : 0u);
    wgmma_commit();
    // keep this stage's MMAs in flight; the previous stage has been read once they are the only ones left
    wgmma_wait<1>();
    __syncwarp();
    if (kb > 0 && lane == 0) mbar_arrive(bar_empty + 8 * ((kb - 1) % kStages));
  }
  wgmma_wait<0>();

  const int rw = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);   // rows rw and rw + 8
  const int cb = n0 + 2 * (lane & 3);                             // columns cb + 8 j + {0, 1}
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = rw + 8 * h;
    if (row >= M) continue;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = cb + 8 * j;
      const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col));
      const float a0 = acc[4 * j + 2 * h] + bb.x, a1 = acc[4 * j + 2 * h + 1] + bb.y;
      const size_t o = (size_t)row * N + col;
      if (EPI == CE_EPI_BIAS_RES_F32) {
        const float2 rb = *reinterpret_cast<const float2*>(residual + o);
        *reinterpret_cast<float2*>(out32 + o) = make_float2(a0 + rb.x, a1 + rb.y);
      } else if (EPI == CE_EPI_BIAS_RES16_F16) {
        const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(reinterpret_cast<const __half*>(residual) + o));
        *reinterpret_cast<__half2*>(out16 + o) = __floats2half2_rn(a0 + rf.x, a1 + rf.y);
      } else {
        *reinterpret_cast<__half2*>(out16 + o) = act_pack<EPI>(a0, a1);
      }
    }
  }
}

template <int EPI>
int launch_gemm(const CUtensorMap& map_a, const CUtensorMap& map_w, int M, int N, int K, const float* bias,
                const float* residual, __half* out16, float* out32, cudaStream_t st, const int* m_dev) {
  static bool configured = false;
  if (!configured) {
    SB_CUDA(cudaFuncSetAttribute(ce_gemm_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemmSmem));
    configured = true;
  }
  const dim3 grid(N / BN, (M + BM - 1) / BM);
  ce_gemm_kernel<EPI><<<grid, kGemmThreads, kGemmSmem, st>>>(map_a, map_w, M, N, K, bias, residual, out16, out32, m_dev);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace

// rows x cols fp16 row-major (cols contiguous) -> 2-D tensor map with a 64 x 128 box and 128-byte swizzle
int ce_make_tensor_map(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols) {
  EncodeTiledFn enc = get_encode();
  SB_REQUIRE(enc != nullptr, SB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  SB_REQUIRE(cols % BK == 0, SB_ERR_ARG, "ce_gemm: K=%lld must be a multiple of %d", (long long)cols, BK);
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SB_REQUIRE(r == CUDA_SUCCESS, SB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return SB_OK;
}

int ce_gemm_launch(int epi, const CUtensorMap& map_a, const CUtensorMap& map_w, int M, int N, int K, const float* bias,
                   const float* residual, __half* out16, float* out32, cudaStream_t st, const int* m_dev) {
  SB_REQUIRE(N % BN == 0 && K % BK == 0, SB_ERR_ARG, "ce_gemm: N=%d / K=%d must be multiples of %d / %d", N, K, BN, BK);
  switch (epi) {
    case CE_EPI_BIAS_F16:
      return launch_gemm<CE_EPI_BIAS_F16>(map_a, map_w, M, N, K, bias, residual, out16, out32, st, m_dev);
    case CE_EPI_BIAS_GELU_F16:
      return launch_gemm<CE_EPI_BIAS_GELU_F16>(map_a, map_w, M, N, K, bias, residual, out16, out32, st, m_dev);
    case CE_EPI_BIAS_RES_F32:
      return launch_gemm<CE_EPI_BIAS_RES_F32>(map_a, map_w, M, N, K, bias, residual, out16, out32, st, m_dev);
    case CE_EPI_BIAS_RES16_F16:
      return launch_gemm<CE_EPI_BIAS_RES16_F16>(map_a, map_w, M, N, K, bias, residual, out16, out32, st, m_dev);
  }
  sb_set_error("ce_gemm: unknown epilogue %d", epi);
  return SB_ERR_ARG;
}
