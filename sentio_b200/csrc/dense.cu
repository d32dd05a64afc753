// dense.cu -- K1: brute-force cosine top-k over an HBM-resident fp16 corpus.
//
// Replaces the Qdrant `client.search(...)` behind DenseRetriever.retrieve (reference src/core/retrievers/dense.py:41-64).
//
// Pipeline per pass of QB (1/2/4) queries:
//   dense_scan_kernel   persistent, one CTA per SM.  A producer warp streams row tiles HBM -> smem with 1-D bulk
//                       async copies (cp.async.bulk, the TMA engine; SASS UBLKCP) through an mbarrier ring; 8 consumer
//                       warps compute fp32 dot products (queries live in registers), apply the stored inverse row norm
//                       and push candidates that beat the CTA's running K'-th best into a smem candidate buffer that
//                       is compacted by an in-smem bitonic sort.  Output: one sorted top-K' list per CTA per query
//                       (K' = k + slack, power of two).
//   dense_merge_kernel  one CTA per query: the k-th best approximate key over the per-CTA lists, then EVERY row inside
//                       the error window below it (dense_common.cuh) is re-scored in fp64 against the STORED fp16 rows,
//                       final sort by (score desc, id asc), write k.  Queries whose window cannot be served from the
//                       lists raise a flag and are answered by dense_exact_fallback_kernel (brute force, fp64).
//
// Algorithmic HBM bytes per pass = n_pad * d_pad * 2 (+ n_pad * 4 for the inverse norms); see DESIGN.md.
#include <float.h>
#include <math.h>
#include <string.h>
#include <algorithm>
#include <cmath>
#include <string>
#include <unordered_map>

#include "dense_common.cuh"
#include "dense_mma.cuh"

namespace {

constexpr int kConsumerWarps = 8;
constexpr int kConsumerThreads = kConsumerWarps * 32;
constexpr int kScanThreads = kConsumerThreads + 64;  // + 1 TMA producer warp + 1 compaction warp
constexpr int kMergeThreads = 512;
constexpr int kRowPad = 128;  // n_pad granularity (tile rows of the wgmma scan; multiple of the CUDA-core tiles)

// ------------------------------------------------------------------------------------------------ load kernels
// One warp per row.  f32 input: x16 = fp16(x / ||x||) (division in fp64, single rounding); f16 input: verbatim.
// inv_norm = 1/||x16|| of the stored values (fp64 accumulate), 0 for all-zero rows.  Input row r goes to row row0 + r,
// or to dst_rows[r] when a destination list is given (sb_dense_upsert).
// Dot / Euclid (cfac != nullptr, always normalised): cfac = c = ||x|| / ||x16|| in fp64 (0 for a zero row), the scan
// scale inv_norm = (float)c, and for Euclid hh = ||v||^2 / 2 = c^2 ||x16||^2 / 2 rounded UP to fp32.
template <typename TIn>
__global__ void dense_store_rows_kernel(const TIn* __restrict__ in, int64_t n_rows, int32_t d, int32_t d_pad,
                                        __half* __restrict__ rows, float* __restrict__ inv_norm, int64_t row0,
                                        const int64_t* __restrict__ dst_rows, bool normalise,
                                        double* __restrict__ cfac, float* __restrict__ hh) {
  int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const int64_t out_row = dst_rows ? dst_rows[r] : row0 + r;
  const TIn* src = in + r * (int64_t)d;
  __half* dst = rows + out_row * (int64_t)d_pad;
  double scale = 1.0;
  if (normalise) {
    double ss = 0.0;
    for (int i = lane; i < d; i += 32) {
      double v = (double)(float)src[i];
      ss += v * v;
    }
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    scale = ss > 0.0 ? sqrt(ss) : 1.0;
  }
  double ss16 = 0.0;
  for (int i = lane; i < d_pad; i += 32) {
    __half h = __float2half(0.f);
    if (i < d) {
      double v = (double)(float)src[i];
      h = normalise ? __double2half(v / scale) : __float2half((float)v);
    }
    dst[i] = h;
    double hv = (double)__half2float(h);
    ss16 += hv * hv;
  }
  for (int o = 16; o; o >>= 1) ss16 += __shfl_xor_sync(0xffffffffu, ss16, o);
  if (lane != 0) return;
  if (cfac == nullptr) {
    inv_norm[out_row] = ss16 > 0.0 ? (float)(1.0 / sqrt(ss16)) : 0.f;
    return;
  }
  const double c = ss16 > 0.0 ? scale / sqrt(ss16) : 0.0;
  cfac[out_row] = c;
  inv_norm[out_row] = (float)c;
  if (hh) hh[out_row] = __double2float_ru(0.5 * (c * c) * ss16);
}

// Float32 storage (DESIGN.md K1g), launched after dense_store_rows_kernel on the same rows: one warp per row writes
// rows32 = x (fp16 input widened exactly, zero padded) and folds the row's sigma into *sigma_bits (an fp64 bit pattern;
// non-negative doubles order like their bits): Cosine ||y/||y|| - x/||x|| ||, Dot / Euclid ||c y - x||, evaluated in
// fp64 and rounded up by the margin DESIGN.md K1g derives.
template <typename TIn>
__global__ void dense_store_rows32_kernel(const TIn* __restrict__ in, int64_t n_rows, int32_t d, int32_t d_pad,
                                          const __half* __restrict__ rows, float* __restrict__ rows32, int64_t row0,
                                          const int64_t* __restrict__ dst_rows, const double* __restrict__ cfac,
                                          unsigned long long* __restrict__ sigma_bits) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const int64_t out_row = dst_rows ? dst_rows[r] : row0 + r;
  const TIn* src = in + r * (int64_t)d;
  const __half* y = rows + out_row * (int64_t)d_pad;
  float* dst = rows32 + out_row * (int64_t)d_pad;
  double xx = 0.0, yy = 0.0;
  for (int i = lane; i < d_pad; i += 32) {
    const float x = i < d ? (float)src[i] : 0.f;
    dst[i] = x;
    const double xd = (double)x, yd = (double)__half2float(y[i]);
    xx = __fma_rn(xd, xd, xx);
    yy = __fma_rn(yd, yd, yy);
  }
  for (int o = 16; o; o >>= 1) {
    xx += __shfl_xor_sync(0xffffffffu, xx, o);
    yy += __shfl_xor_sync(0xffffffffu, yy, o);
  }
  const double nx = sqrt(xx), ny = sqrt(yy);
  const double c = cfac ? cfac[out_row] : 0.0;
  double ee = 0.0;
  for (int i = lane; i < d; i += 32) {
    const double xd = (double)(float)src[i], yd = (double)__half2float(y[i]);
    const double t = cfac ? __fma_rn(c, yd, -xd) : __dsub_rn(ny > 0.0 ? yd / ny : 0.0, nx > 0.0 ? xd / nx : 0.0);
    ee = __fma_rn(t, t, ee);
  }
  for (int o = 16; o; o >>= 1) ee += __shfl_xor_sync(0xffffffffu, ee, o);
  if (lane != 0) return;
  const double m = cfac ? nx : 1.0;
  const double sig = __fma_ru(sqrt(ee), 1.0 + 0x1p-39, m * 0x1p-39);
  atomicMax(sigma_bits, (unsigned long long)__double_as_longlong(sig));
}

// Uint8 storage (DESIGN.md K1i): one warp per row writes rows8 = x (zero padded to d_pad bytes), the scan scale inv_norm
// (Cosine fl32(1/||x||), 0 for a zero row; Dot / Euclid 1: the scan reads x itself), for Euclid hh = ||x||^2 / 2 rounded
// up to fp32, and folds the row's ||x||^2 (an integer below 2^28) into *xx_max.  The host has checked that every input
// value is an integer in [0, 255].
template <typename TIn>
__global__ void dense_store_rows8_kernel(const TIn* __restrict__ in, int64_t n_rows, int32_t d, int32_t d_pad,
                                         uint8_t* __restrict__ rows8, float* __restrict__ inv_norm, int64_t row0,
                                         const int64_t* __restrict__ dst_rows, bool cosine, float* __restrict__ hh,
                                         unsigned long long* __restrict__ xx_max) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const int64_t out_row = dst_rows ? dst_rows[r] : row0 + r;
  const TIn* src = in + r * (int64_t)d;
  uint8_t* dst = rows8 + out_row * (int64_t)d_pad;
  uint32_t ss = 0;
  for (int i = lane; i < d_pad; i += 32) {
    const uint32_t v = i < d ? (uint32_t)(float)src[i] : 0u;
    dst[i] = (uint8_t)v;
    ss += v * v;
  }
  for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane != 0) return;
  inv_norm[out_row] = cosine ? (ss ? (float)(1.0 / sqrt((double)ss)) : 0.f) : 1.f;
  if (hh) hh[out_row] = __double2float_ru(0.5 * (double)ss);
  atomicMax(xx_max, (unsigned long long)ss);
}

// ------------------------------------------------------------------------------------------------ mutation kernels
// sb_dense_delete's compaction: one warp per move from[m] -> to[m] (sources >= n - |D| > destinations, so one launch
// has no read/write hazard) copies the row in every column of the slot (dense_columns): a row that is a multiple of
// 16 bytes (the vectors) in 16-byte copies spread over the lanes, a 4- or 8-byte row by one lane.
constexpr int kMaxDenseColumns = 5 + SB_MAX_TAG_FIELDS + SB_MAX_VALUE_FIELDS;

struct MoveParams {
  uint8_t* col[kMaxDenseColumns];
  int32_t row_bytes[kMaxDenseColumns];
  int32_t n_cols;
  const int64_t* from;
  const int64_t* to;
  int64_t n_moves;
};

__global__ void __launch_bounds__(256, 8) dense_move_rows_kernel(const __grid_constant__ MoveParams p) {
  const int64_t m = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (m >= p.n_moves) return;
  const int64_t s = p.from[m], t = p.to[m];
  for (int c = 0; c < p.n_cols; ++c) {
    const int rb = p.row_bytes[c];
    if (rb % 16) continue;
    const uint4* src = reinterpret_cast<const uint4*>(p.col[c] + s * rb);
    uint4* dst = reinterpret_cast<uint4*>(p.col[c] + t * rb);
#pragma unroll 4   // the default unroll spills
    for (int i = lane; i < rb / 16; i += 32) dst[i] = src[i];
  }
  for (int c = lane; c < p.n_cols; c += 32) {
    const int rb = p.row_bytes[c];
    if (rb == 8) reinterpret_cast<uint64_t*>(p.col[c])[t] = reinterpret_cast<const uint64_t*>(p.col[c])[s];
    else if (rb == 4) reinterpret_cast<uint32_t*>(p.col[c])[t] = reinterpret_cast<const uint32_t*>(p.col[c])[s];
  }
}

// codes[i] -> col[rows[i]]; codes == nullptr writes -1 (an upserted row's payload is unknown until its codes arrive)
__global__ void __launch_bounds__(256) dense_tags_scatter_kernel(int32_t* __restrict__ col,
                                                                 const int64_t* __restrict__ rows,
                                                                 const int32_t* __restrict__ codes, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) col[rows[i]] = codes ? codes[i] : -1;
}

// vals[i] -> col[rows[i]]; vals == nullptr writes NaN (all bits set, the pattern of unused capacity)
__global__ void __launch_bounds__(256) dense_values_scatter_kernel(double* __restrict__ col,
                                                                   const int64_t* __restrict__ rows,
                                                                   const double* __restrict__ vals, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) col[rows[i]] = vals ? vals[i] : __longlong_as_double(-1ll);
}

// ------------------------------------------------------------------------------------------------ scan kernel
struct ScanParams {
  const __half* rows;
  const float* inv_norm;
  const float* q;            // [QB][d_pad] fp32 (zero padded) for THIS pass
  unsigned long long* cand;  // [QB][grid][kprime] composite keys, sorted descending per list
  int64_t n;                 // valid rows
  int32_t d_pad;
  int32_t ch;                // 16-byte chunks per row = d_pad / 8
  int32_t num_tiles;
  int32_t kprime;
  int32_t bcap;              // capacity of each of the two append batches per query (kprime + bcap = sort size)
  int32_t stages;
  uint32_t tile_bytes;
  // FILTER only: match bits of this pass's queries (bit r % 32 of mask[(r / 32) * mask_qs + query]) and the per-query
  // state (1 = answered by the gather path: threshold +inf, nothing is appended)
  const uint32_t* mask;
  int32_t mask_qs;
  const int32_t* state;
  // EUCLID only: per-row h (>= ||v||^2 / 2) and per-query r = (float)||q|| of this pass's queries
  const float* hh;
  const float* rq;
};

// Sum V per-lane partials across the warp: afterwards the lanes with (lane % (32/V)) == 0 hold value index lane/(32/V).
template <int V>
__device__ __forceinline__ float warp_reduce_multi(float (&v)[V], int lane) {
  int off = 16;
#pragma unroll
  for (int half = V / 2; half >= 1; half >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int t = 0; t < half; ++t) {
      float send = upper ? v[t] : v[t + half];
      float keep = upper ? v[t + half] : v[t];
      v[t] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
    off >>= 1;
  }
  float r = v[0];
  for (; off >= 1; off >>= 1) r += __shfl_xor_sync(0xffffffffu, r, off);
  return r;
}

// ---- asynchronous compaction (runs on its own warp, off the FMA warps' critical path) -------------------------------
// Descending bitonic sort of T = 32 * NPER 64-bit keys held in registers across one warp; element e = lane * NPER + r.
template <int NPER>
__device__ __forceinline__ void warp_sort_desc(unsigned long long (&v)[NPER], int lane) {
  constexpr int T = NPER * 32;
#pragma unroll
  for (int k = 2; k <= T; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j < NPER) {
#pragma unroll
        for (int r = 0; r < NPER; ++r) {
          const int pr = r ^ j;
          if (pr > r) {
            const bool desc = (k < NPER) ? ((r & k) == 0) : ((lane & (k / NPER)) == 0);
            const unsigned long long x = v[r], y = v[pr];
            const bool sw = desc ? (x < y) : (x > y);
            v[r] = sw ? y : x;
            v[pr] = sw ? x : y;
          }
        }
      } else {
        const int lj = j / NPER;
        const bool lower = (lane & lj) == 0;
        const bool desc = (lane & (k / NPER)) == 0;
        const bool keep_max = lower == desc;
#pragma unroll
        for (int r = 0; r < NPER; ++r) {
          const unsigned long long o = __shfl_xor_sync(0xffffffffu, v[r], lj);
          const unsigned long long x = v[r];
          v[r] = keep_max ? (x > o ? x : o) : (x < o ? x : o);
        }
      }
    }
  }
}

// best[0..nbest) U batch[0..nbatch)  ->  best[0..min(K', nbest+nbatch))  (sorted descending); returns the new count.
template <int NPER>
__device__ __noinline__ int compact_into_best(unsigned long long* best, int nbest, const unsigned long long* batch,
                                              int nbatch, int kprime, int lane) {
  unsigned long long v[NPER];
#pragma unroll
  for (int r = 0; r < NPER; ++r) {
    const int e = lane * NPER + r;
    unsigned long long x = 0ull;
    if (e < nbest) x = best[e];
    else if (e - nbest < nbatch) x = batch[e - nbest];
    v[r] = x;
  }
  __syncwarp();
  warp_sort_desc<NPER>(v, lane);
#pragma unroll
  for (int r = 0; r < NPER; ++r) {
    const int e = lane * NPER + r;
    if (e < kprime) best[e] = v[r];
  }
  __syncwarp();
  const int total = nbest + nbatch;
  return total < kprime ? total : kprime;
}

// Generic (k > 100) path: same result through a shared-memory scratch of T keys, loop-based warp bitonic sort.
__device__ __noinline__ int compact_into_best_smem(unsigned long long* best, int nbest, const unsigned long long* batch,
                                                   int nbatch, int kprime, int T, unsigned long long* scratch,
                                                   int lane) {
  for (int e = lane; e < T; e += 32) {
    unsigned long long x = 0ull;
    if (e < nbest) x = best[e];
    else if (e - nbest < nbatch) x = batch[e - nbest];
    scratch[e] = x;
  }
  __syncwarp();
  for (int k = 2; k <= T; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < T; i += 32) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long x = scratch[i], y = scratch[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? (x < y) : (x > y)) {
            scratch[i] = y;
            scratch[ixj] = x;
          }
        }
      }
      __syncwarp();
    }
  }
  for (int e = lane; e < kprime; e += 32) best[e] = scratch[e];
  __syncwarp();
  const int total = nbest + nbatch;
  return total < kprime ? total : kprime;
}

__device__ __forceinline__ int compact_dispatch(int T, unsigned long long* best, int nbest,
                                                const unsigned long long* batch, int nbatch, int kprime,
                                                unsigned long long* scratch, int lane) {
  if (T == 512) return compact_into_best<16>(best, nbest, batch, nbatch, kprime, lane);
  return compact_into_best_smem(best, nbest, batch, nbatch, kprime, T, scratch, lane);
}

// a (lo, hi) pair of fp32 FMAs on floats packed in 64-bit registers: two FFMA on sm_90 (full rate there), each lane
// rounded exactly as one fma.rn
__device__ __forceinline__ unsigned long long ffma2(unsigned long long a, unsigned long long b, unsigned long long c) {
  const float lo = fmaf(__uint_as_float((uint32_t)a), __uint_as_float((uint32_t)b), __uint_as_float((uint32_t)c));
  const float hi = fmaf(__uint_as_float((uint32_t)(a >> 32)), __uint_as_float((uint32_t)(b >> 32)),
                        __uint_as_float((uint32_t)(c >> 32)));
  return ((unsigned long long)__float_as_uint(hi) << 32) | (unsigned long long)__float_as_uint(lo);
}
__device__ __forceinline__ unsigned long long pack_f2(float lo, float hi) {
  return ((unsigned long long)__float_as_uint(hi) << 32) | (unsigned long long)__float_as_uint(lo);
}
__device__ __forceinline__ unsigned long long h2_to_f2(uint32_t h2) {
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h2));
  return pack_f2(f.x, f.y);
}

// Key of a row: Cosine / Dot  acc * scale[row];  EUCLID  r * (acc * scale[row]) - h[row] = (||q||^2 - ||q - v||^2) / 2
// up to the error bound of DESIGN.md K1e (larger = nearer).
template <int NCHUNK, int QB, int RW, bool EXACT, bool FILTER, bool EUCLID>
__global__ void __launch_bounds__(kScanThreads, 1) dense_scan_kernel(const ScanParams p) {
  constexpr int R = kConsumerWarps * RW;  // rows per tile
  constexpr int V = RW * QB;              // partial sums per lane
  constexpr int LPV = 32 / V;             // lanes per value after the reduction
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* tiles = smem;
  // per query: best[K'] (sorted, owned by the compaction warp) + two append batches of bcap keys (ping / pong)
  const int qstride = p.kprime + 2 * p.bcap;
  unsigned long long* cbuf = reinterpret_cast<unsigned long long*>(smem + (size_t)p.stages * p.tile_bytes);
  const int scratch_keys = (p.kprime + p.bcap == 512) ? 0 : (p.kprime + p.bcap);
  unsigned long long* bars = cbuf + (size_t)QB * qstride + scratch_keys;  // full[stages], empty[stages]
  volatile int* cnt = reinterpret_cast<volatile int*>(bars + 2 * p.stages);        // [QB][2] appended per batch
  volatile float* thr = reinterpret_cast<volatile float*>(const_cast<int*>(cnt) + 2 * QB);
  volatile int* active = reinterpret_cast<volatile int*>(const_cast<float*>(thr) + QB);   // [QB] batch being appended
  volatile int* pending = active + QB;   // [QB] 0 = idle, 1 = batch (1 - active) waits for compaction
  volatile int* frozen = pending + QB;   // [QB] entry count of the batch handed to the compaction warp
  volatile int* nbest = frozen + QB;     // [QB]
  volatile int* done_flag = nbest + QB;  // [1] consumers finished streaming

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int stages = p.stages;
  const uint32_t bar_full0 = smem_u32(bars), bar_empty0 = smem_u32(bars + stages);

  if (tid == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(bar_full0 + 8 * s, 1);
      mbar_init(bar_empty0 + 8 * s, kConsumerWarps);
    }
    mbar_fence_init();
  }
  if (tid < QB) {
    cnt[2 * tid] = 0;
    cnt[2 * tid + 1] = 0;
    if constexpr (FILTER) thr[tid] = p.state[tid] ? INFINITY : -INFINITY;
    else thr[tid] = -INFINITY;
    active[tid] = 0;
    pending[tid] = 0;
    frozen[tid] = 0;
    nbest[tid] = 0;
  }
  if (tid == 0) done_flag[0] = 0;
  __syncthreads();

  const int grid = gridDim.x;
  const int my_tiles = ((int)blockIdx.x < p.num_tiles) ? (p.num_tiles - 1 - (int)blockIdx.x) / grid + 1 : 0;
  const uint32_t row_bytes = (uint32_t)p.d_pad * 2u;

  if (warp == kConsumerWarps) {
    // ------------------------------------------------------------ producer warp: one elected lane drives the TMA ring
    if (lane == 0) {
      const uint64_t policy = policy_evict_first();
      const uint32_t tiles_s = smem_u32(tiles);
      for (int i = 0; i < my_tiles; ++i) {
        const int s = i % stages;
        const uint32_t use = (uint32_t)(i / stages);
        if (i >= stages) mbar_wait(bar_empty0 + 8 * s, (use & 1u) ^ 1u);
        const int64_t tile = (int64_t)blockIdx.x + (int64_t)i * grid;
        const uint8_t* src = reinterpret_cast<const uint8_t*>(p.rows) + (size_t)tile * p.tile_bytes;
        mbar_expect_tx(bar_full0 + 8 * s, p.tile_bytes);
        bulk_g2s(tiles_s + (uint32_t)s * p.tile_bytes, src, p.tile_bytes, bar_full0 + 8 * s, policy);
      }
    }
    return;
  }

  if (warp == kConsumerWarps + 1) {
    // ------------------------------------------------------------ compaction warp: folds full batches into best[],
    // publishes the rising threshold, and emits the final sorted top-K' lists.  Never blocks the FMA warps.
    const int T = p.kprime + p.bcap;
    unsigned long long* scratch = cbuf + (size_t)QB * qstride;  // only present when T != 512
    for (;;) {
      const bool fin = done_flag[0] != 0;
      __threadfence_block();
      bool any = false;
      for (int q = 0; q < QB; ++q) {
        if (pending[q]) {
          __threadfence_block();
          unsigned long long* best = cbuf + (size_t)q * qstride;
          const unsigned long long* batch = best + p.kprime + (size_t)(1 - active[q]) * p.bcap;
          const int nb = compact_dispatch(T, best, nbest[q], batch, frozen[q], p.kprime, scratch, lane);
          if (lane == 0) {
            nbest[q] = nb;
            if (nb >= p.kprime) thr[q] = key32_score(best[p.kprime - 1]);
            __threadfence_block();
            pending[q] = 0;
          }
          __syncwarp();
          any = true;
        }
      }
      if (fin && !any) break;
      if (!any) __nanosleep(200);
    }
    // final: fold the batch still being appended, then write the sorted list of every query
    for (int q = 0; q < QB; ++q) {
      unsigned long long* best = cbuf + (size_t)q * qstride;
      const int a = active[q];
      const unsigned long long* batch = best + p.kprime + (size_t)a * p.bcap;
      const int nb = compact_dispatch(T, best, nbest[q], batch, min((int)cnt[2 * q + a], p.bcap), p.kprime, scratch, lane);
      unsigned long long* out = p.cand + ((size_t)q * grid + blockIdx.x) * p.kprime;
      for (int z = lane; z < p.kprime; z += 32) out[z] = z < nb ? best[z] : 0ull;
    }
    return;
  }

  // -------------------------------------------------------------- consumer warps
  // query slices in registers as (even, odd) fp32 pairs: lane owns 16-byte chunk c = lane + 32*j of every row
  unsigned long long qr[QB][NCHUNK][4];
#pragma unroll
  for (int q = 0; q < QB; ++q) {
#pragma unroll
    for (int j = 0; j < NCHUNK; ++j) {
      const int c = lane + 32 * j;
      if (EXACT || c < p.ch) {
        const float4* src = reinterpret_cast<const float4*>(p.q + (size_t)q * p.d_pad + (size_t)c * 8);
        const float4 a = __ldg(src), b = __ldg(src + 1);
        qr[q][j][0] = pack_f2(a.x, a.y);
        qr[q][j][1] = pack_f2(a.z, a.w);
        qr[q][j][2] = pack_f2(b.x, b.y);
        qr[q][j][3] = pack_f2(b.z, b.w);
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) qr[q][j][e] = 0ull;
      }
    }
  }

  const int vi = lane / LPV;          // which (row, query) this lane owns after the reduction
  const int ri = vi / QB, qi = vi % QB;
  const bool leader = (lane % LPV) == 0;
  const int trigger = p.bcap - R;  // a batch is handed over while it still has room for one more tile
  float rq = 0.f;
  if constexpr (EUCLID) rq = __ldg(p.rq + qi);

  for (int i = 0; i < my_tiles; ++i) {
    const int s = i % stages;
    const uint32_t use = (uint32_t)(i / stages);
    const int64_t tile = (int64_t)blockIdx.x + (int64_t)i * grid;
    const int64_t grow = tile * R + warp * RW + ri;
    mbar_wait(bar_full0 + 8 * s, use & 1u);
    float invn = 0.f;
    if (leader) invn = __ldg(p.inv_norm + grow);  // consumed after the reduction: latency hides under the FMAs
    float hrow = 0.f;
    if constexpr (EUCLID)
      if (leader) hrow = __ldg(p.hh + grow);
    uint32_t mword = 0u;
    if constexpr (FILTER)
      if (leader) mword = __ldg(p.mask + (size_t)(grow >> 5) * p.mask_qs + qi);

    unsigned long long acc[V];
#pragma unroll
    for (int v = 0; v < V; ++v) acc[v] = 0ull;
    const uint8_t* wbase = tiles + (size_t)s * p.tile_bytes + (size_t)(warp * RW) * row_bytes + (size_t)lane * 16;
    // software pipeline at (chunk, row) granularity: the 16 bytes of the next step are in flight while this step is
    // converted and multiplied (one uint4 of look-ahead keeps the register budget under the 200-register ceiling)
    uint4 cur = make_uint4(0u, 0u, 0u, 0u);
    if (EXACT || lane < p.ch) cur = *reinterpret_cast<const uint4*>(wbase);
#pragma unroll
    for (int step = 0; step < NCHUNK * RW; ++step) {
      const int j = step / RW, r = step % RW;
      uint4 nxt = make_uint4(0u, 0u, 0u, 0u);
      if (step + 1 < NCHUNK * RW) {
        const int jn = (step + 1) / RW, rn = (step + 1) % RW;
        if (EXACT || lane + 32 * jn < p.ch)
          nxt = *reinterpret_cast<const uint4*>(wbase + (size_t)rn * row_bytes + (size_t)jn * 512);
      }
      const unsigned long long x0 = h2_to_f2(cur.x), x1 = h2_to_f2(cur.y);
      const unsigned long long x2 = h2_to_f2(cur.z), x3 = h2_to_f2(cur.w);
#pragma unroll
      for (int q = 0; q < QB; ++q) {
        unsigned long long a = acc[r * QB + q];
        a = ffma2(x0, qr[q][j][0], a);
        a = ffma2(x1, qr[q][j][1], a);
        a = ffma2(x2, qr[q][j][2], a);
        a = ffma2(x3, qr[q][j][3], a);
        acc[r * QB + q] = a;
      }
      cur = nxt;
    }
    // all smem reads of this stage are consumed (their values fed the FMAs above) -> release the slot
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty0 + 8 * s);

    float part[V];
#pragma unroll
    for (int v = 0; v < V; ++v)
      part[v] = __uint_as_float((uint32_t)(acc[v] & 0xffffffffull)) + __uint_as_float((uint32_t)(acc[v] >> 32));
    const float dot = warp_reduce_multi<V>(part, lane);
    if (leader) {
      float score = dot * invn;
      if constexpr (EUCLID) score = __fsub_rn(__fmul_rn(rq, score), hrow);
      bool match = true;
      if constexpr (FILTER) match = (mword >> (grow & 31)) & 1u;
      if (grow < p.n && score > thr[qi] && match) {
        const int a = active[qi];
        const int pos = atomicAdd(const_cast<int*>(&cnt[2 * qi + a]), 1);
        if (pos < p.bcap) cbuf[(size_t)qi * qstride + p.kprime + (size_t)a * p.bcap + pos] = make_key32(score, (uint32_t)grow);
      }
    }
    bool need = false;
#pragma unroll
    for (int q = 0; q < QB; ++q) need |= (cnt[2 * q + active[q]] > trigger);
    need = named_bar_or(2, kConsumerThreads, need);
    if (need) {
      // hand the nearly full batch of every such query to the compaction warp and continue on the other batch
      if (tid == 0) {
        for (int q = 0; q < QB; ++q) {
          const int a = active[q];
          const int c = cnt[2 * q + a];
          if (c > trigger) {
            while (pending[q]) __nanosleep(64);  // previous hand-over still being folded (practically never)
            __threadfence_block();
            frozen[q] = min(c, p.bcap);
            cnt[2 * q + (1 - a)] = 0;
            active[q] = 1 - a;
            __threadfence_block();
            pending[q] = 1;
          }
        }
      }
      named_bar_sync(1, kConsumerThreads);
    }
  }

  // -------------------------------------------------------------- streaming finished: the compaction warp finalises
  named_bar_sync(1, kConsumerThreads);
  if (tid == 0) {
    __threadfence_block();
    done_flag[0] = 1;
  }
}

// ------------------------------------------------------------------------------------------------ merge kernel
constexpr int kSelCap = 2048;  // shared-memory capacity of the window (winner) set

struct MergeParams {
  const unsigned long long* cand;  // [nq][G][kprime] sorted descending lists
  int32_t G;
  int32_t kprime;
  int32_t heads_per_list;    // R = ceil(kprime / G)
  int32_t heads_pow2;        // power of two >= G * R  (<= kSelCap)
  SlotView slot;
  const float* q;            // [nq][d_pad] the caller's fp32 queries (exact stage)
  const float* eps;          // [nq] error bound of the approximate scores (0 for an all-zero query)
  int32_t* fallback;         // [nq] raised when the lists cannot serve the window
  int32_t k;
  int64_t* out_ids;          // [nq][k]
  double* out_scores;        // [nq][k]
  int32_t* out_counts;       // [nq]
  const int32_t* state;      // FILTER only: [nq] 1 = answered by the gather path (nothing to merge)
};

__device__ __forceinline__ void block_sort_desc_u64(unsigned long long* a, int len, int tid, int nt) {
  for (int k = 2; k <= len; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < len; i += nt) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long x = a[i], y = a[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? (x < y) : (x > y)) {
            a[i] = y;
            a[ixj] = x;
          }
        }
      }
      __syncthreads();
    }
  }
}

// One CTA per query.  (1) a lower bound of the global k-th best approximate key = the k-th largest among the first
// R = ceil(K'/G) entries of every list (G*R >= K' >= k real keys); (2) every list contributes its prefix inside the
// error window below that key; a FULL list whose last entry is still inside the window may have dropped members ->
// fallback; (3) exact fp64 re-score of the whole window (F32: against the float32 rows); (4) final order, emit k.
template <bool FILTER, bool F32>
__global__ void __launch_bounds__(kMergeThreads, 1) dense_merge_kernel(const MergeParams p) {
  extern __shared__ __align__(16) uint8_t msmem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x, nw = nt >> 5;
  const int qi = blockIdx.x;
  if constexpr (FILTER)
    if (p.state[qi]) return;
  const int G = p.G, K = p.kprime;
  unsigned long long* sel = reinterpret_cast<unsigned long long*>(msmem);   // [kSelCap]
  unsigned long long* ek = sel + kSelCap;                                   // [kSelCap] exact score keys
  uint32_t* ei = reinterpret_cast<uint32_t*>(ek + kSelCap);                 // [kSelCap] row index
  float* q_s = reinterpret_cast<float*>(ei + kSelCap);                      // [d_pad]   the query, staged once
  __shared__ double qq_s;
  __shared__ int s_nsel, s_trunc;
  __shared__ unsigned long long s_bound;
  const unsigned long long* L = p.cand + (size_t)qi * G * K;

  // (1) bound from the list heads
  const int R = p.heads_per_list, nh = G * R, HP = p.heads_pow2;
  for (int t = tid; t < HP; t += nt) sel[t] = t < nh ? L[(size_t)(t / R) * K + (t % R)] : 0ull;
  if (tid == 0) {
    s_nsel = 0;
    s_trunc = 0;
  }
  __syncthreads();
  block_sort_desc_u64(sel, HP, tid, nt);
  // fewer than k rows in the whole corpus -> sel[k-1] is an empty slot (0): everything is a member
  if (tid == 0) s_bound = sel[p.k - 1] != 0ull ? window_lo_key(sel[p.k - 1], p.eps[qi]) : 0ull;
  __syncthreads();
  const unsigned long long bound = s_bound;
  __syncthreads();  // sel is reused below

  // (2) gather every list's prefix >= bound (lists are sorted descending; empty slots are key 0)
  for (int g = warp; g < G; g += nw) {
    const unsigned long long* lst = L + (size_t)g * K;
    for (int base = 0; base < K; base += 32) {
      const unsigned long long key = lst[base + lane];
      const bool pass = key >= bound && key != 0ull;
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      if (m == 0u) break;
      int pos = 0;
      if (lane == 0) pos = atomicAdd(&s_nsel, __popc(m));
      pos = __shfl_sync(0xffffffffu, pos, 0);
      if (pass) {
        const int at = pos + __popc(m & ((1u << lane) - 1u));
        if (at < kSelCap) sel[at] = key;
      }
      if (m != 0xffffffffu) break;
      if (base + 32 >= K && lane == 0) s_trunc = 1;  // the whole (full) list is inside the window
    }
  }
  __syncthreads();
  const int nsel = s_nsel;
  if (nsel > kSelCap || s_trunc) {
    if (tid == 0) p.fallback[qi] = 1;
    return;
  }
  int P = 32;
  while (P < nsel) P <<= 1;

  const RescoreArgs ra{p.slot, p.q + (size_t)qi * p.slot.d_pad, p.k, p.out_ids + (size_t)qi * p.k,
                       p.out_scores + (size_t)qi * p.k, p.out_counts + qi};
  rescore_and_emit<F32 ? SB_STORAGE_F32 : SB_STORAGE_F16>(sel, nsel, P, ek, ei, &qq_s, q_s, ra);
}

// ------------------------------------------------------------------------------------------------ query preparation
// One CTA per operand row r (rows >= nq are padding): qn[r] = q[r] / ||q[r]|| in fp32 (the scans rank by cosine, so the
// caller's scale must not reach the fp32 / fp16 arithmetic), optionally q16[r] = fp16(qn[r]) for the wgmma scan, and
// eps[r] = the bound on |approximate - exact cosine| the hand-off window uses (0 for an all-zero query).
// Dot / Euclid (DESIGN.md K1e): eps[r] bounds |approximate - exact key| in key units, from the cosine bound and the slot's
// norm bounds rho (>= max ||v||) and hmax (>= max h); Euclid also writes rq[r] = (float)||q[r]||.  A query whose key
// could leave the fp32 range, or whose exact fp64 distances cannot resolve the window, gets its fallback flag fb[r].
// Float32 storage (DESIGN.md K1g) adds sigma (>= ||y^ - x^|| resp. ||v - x|| over the slot's rows): the key of x differs
// from the key of v by at most sigma (Cosine, Dot) or (r + rho) sigma (Euclid); sigma = 0 for float16 storage.
// Uint8 storage (DESIGN.md K1i): the scan reads x itself, so sigma = 0 and rho, hmax bound ||x|| and ||x||^2 / 2.  q16 is
// written with its columns permuted inside every 64-column block (u8_query_column), so that the 16 bytes a scan thread
// reads from a corpus row are its wgmma A fragments for the block's four k16 steps.
struct PrepMetric {
  int32_t metric;
  double rho, hmax, sigma;
  float* rq;      // [rows] Euclid
  int32_t* fb;    // [rows]
};

template <int ST>
__global__ void __launch_bounds__(256) dense_prep_queries_kernel(const float* __restrict__ q_pad, int nq, int d_pad,
                                                                 float* __restrict__ qn, __half* __restrict__ q16,
                                                                 float* __restrict__ eps, int mma, const PrepMetric pm) {
  __shared__ double s_red[8];
  __shared__ double s_tot;
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool real = r < nq;
  const float* src = q_pad + (size_t)r * d_pad;
  double ss = 0.0;
  if (real)
    for (int i = tid; i < d_pad; i += blockDim.x) {
      const double v = (double)src[i];
      ss += v * v;
    }
  for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) s_red[warp] = ss;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
    s_tot = t;
  }
  __syncthreads();
  const double nrm = sqrt(s_tot);
  const bool zero = !(nrm > 0.0) || !real;
  if (pm.rq && tid == 0) pm.rq[r] = zero ? 0.f : (float)nrm;
  double dd = 0.0;  // ||fp16(qn) - qn||^2
  for (int i = tid; i < d_pad; i += blockDim.x) {
    const float v = zero ? 0.f : (float)((double)src[i] / nrm);
    if (qn) qn[(size_t)r * d_pad + i] = v;
    if (q16) {
      const __half h = __float2half_rn(v);
      if constexpr (ST == SB_STORAGE_U8) q16[(size_t)r * d_pad + (i & ~63) + u8_query_column(i & 63)] = h;
      else q16[(size_t)r * d_pad + i] = h;
      const double e = (double)__half2float(h) - (double)v;
      dd += e * e;
    }
  }
  if (eps == nullptr || !real) return;
  for (int o = 16; o; o >>= 1) dd += __shfl_xor_sync(0xffffffffu, dd, o);
  __syncthreads();
  if (lane == 0) s_red[warp] = dd;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
    float e = 0.f;
    if (!zero) e = mma ? (float)(sqrt(t) * 1.0001) + dense_eps_mma_acc(d_pad) : dense_eps_fp32(d_pad);
    // float32 storage (DESIGN.md K1g): + sigma (Cosine, Dot), + (r + rho) sigma (Euclid), the first through r * ed
    if constexpr (ST == SB_STORAGE_F32)
      if (pm.metric == SB_METRIC_COSINE && !zero) e = __double2float_ru((double)e + pm.sigma);
    if (pm.metric != SB_METRIC_COSINE) {
      // Dot: |acc * (float)c - <qn, v>| <= c (e + 2^-22) with c <= rho (1 + 2^-10); the zero query keeps eps 0 (every key
      // is exactly 0).  Euclid: key = r * (acc * s) - h; r * eps_dot + r rho 2^-22 (r and its product) + hmax 2^-22 (h
      // rounded up) + (r rho + hmax) 2^-24 (the subtraction), all inside (r rho + hmax) 2^-20.
      double ed = ((double)e + 0x1p-20) * pm.rho * 1.001;
      if constexpr (ST == SB_STORAGE_F32) ed += pm.sigma;
      const bool fits = pm.rho <= 1e36;
      if (pm.metric == SB_METRIC_DOT) {
        e = zero ? 0.f : __double2float_ru(ed);
        if (!fits) pm.fb[r] = 1;
      } else {
        const double rr = zero ? 0.0 : (double)(float)nrm;
        double ee = (rr * ed + (rr * pm.rho + pm.hmax) * 0x1p-20) * 1.001;
        if constexpr (ST == SB_STORAGE_F32) ee += pm.rho * pm.sigma * 1.001;   // | ||v||^2 - ||x||^2 | / 2 <= (rho + sigma / 2) sigma
        e = __double2float_ru(ee);
        // the fp64 exact stage resolves ||q - v||^2 to (r + rho)^2 2^-41 (d <= 4096 terms); it must stay far below eps
        const double res = (rr + pm.rho) * (rr + pm.rho) * 0x1p-41;
        if (!(rr * pm.rho <= 1e36 && pm.hmax <= 1e36 && fits && res * 1024.0 <= ee)) pm.fb[r] = 1;
      }
    }
    eps[r] = e;
  }
}

// ------------------------------------------------------------------------------------------------ exact fallback
// One CTA per FLAGGED query (the others exit at once): brute force over every stored row in fp64 -- 1024 rows per round
// are scored by the CTA's 32 warps and folded into the running best list by a 2048-pair bitonic sort (skipped when no
// new row beats the current k-th best).  Slow (tens of ms at 1 M rows) and exact for any score distribution.
constexpr int kFbThreads = 1024;
constexpr int kFbBest = 1024;  // >= the largest supported k

struct FallbackParams {
  const int32_t* flag;   // [nq]
  SlotView slot;
  const float* q;        // [nq][d_pad]
  int64_t n;
  int32_t k;
  int64_t* out_ids;
  double* out_scores;
  int32_t* out_counts;
  unsigned long long* counter;   // [1] queries answered here since the context was created
  const uint32_t* mask;          // FILTER only: match bits, mask[(row / 32) * mask_qs + query]
  int32_t mask_qs;
};

template <bool FILTER, int ST>
__global__ void __launch_bounds__(kFbThreads, 1) dense_exact_fallback_kernel(const FallbackParams p) {
  const int qi = blockIdx.x;
  if (p.flag[qi] == 0) return;
  __shared__ unsigned long long ek[2 * kFbBest];
  __shared__ uint32_t ei[2 * kFbBest];
  __shared__ double qq_s;
  __shared__ int s_beats;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x, nw = nt >> 5;
  if (tid == 0) atomicAdd(p.counter, 1ull);
  const float* q = p.q + (size_t)qi * p.slot.d_pad;
  const double qn = query_norm_cta(q, p.slot.d_pad, &qq_s);
  // Cosine / Dot: the all-zero query scores 0 on every row.  Euclid: it does not (the nearest rows are the smallest).
  const bool zero_shortcut = !(qn > 0.0) && p.slot.metric != SB_METRIC_EUCLID;
  if (FILTER && zero_shortcut) {
    // all-zero query: every cosine is 0 -> the first k MATCHING rows in index order (one warp walks the mask words)
    if (warp != 0) return;
    const int64_t n_words = (p.n + 31) / 32;
    int got = 0;
    for (int64_t w0 = 0; w0 < n_words && got < p.k; w0 += 32) {
      const int64_t w = w0 + lane;
      uint32_t bits = w < n_words ? p.mask[(size_t)w * p.mask_qs + qi] : 0u;
      const int c = __popc(bits);
      int incl = c;
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      for (int pos = got + incl - c; bits != 0u && pos < p.k; ++pos) {
        const int b = __ffs(bits) - 1;
        bits &= bits - 1u;
        p.out_ids[(size_t)qi * p.k + pos] = p.slot.id_base + w * 32 + b;
        p.out_scores[(size_t)qi * p.k + pos] = 0.0;
      }
      got += __shfl_sync(0xffffffffu, incl, 31);
    }
    const int m = min(got, p.k);
    for (int i = m + lane; i < p.k; i += 32) {
      p.out_ids[(size_t)qi * p.k + i] = -1;
      p.out_scores[(size_t)qi * p.k + i] = 0.0;
    }
    if (lane == 0) p.out_counts[qi] = m;
    return;
  }
  if (zero_shortcut) {
    // all-zero query: every cosine is exactly 0 -> the first k rows in index order, no scan needed
    const int m = (int)min((int64_t)p.k, p.n);
    for (int i = tid; i < p.k; i += nt) {
      p.out_ids[(size_t)qi * p.k + i] = i < m ? p.slot.id_base + i : -1;
      p.out_scores[(size_t)qi * p.k + i] = 0.0;
    }
    if (tid == 0) p.out_counts[qi] = m;
    return;
  }
  for (int i = tid; i < 2 * kFbBest; i += nt) {
    ek[i] = 0ull;
    ei[i] = 0xffffffffu;
  }
  __syncthreads();
  for (int64_t r0 = 0; r0 < p.n; r0 += kFbBest) {
    if (tid == 0) s_beats = 0;
    __syncthreads();
    const unsigned long long kth = ek[p.k - 1];  // 0 while fewer than k rows have been seen
    bool beat = false;
    for (int c = warp; c < kFbBest; c += nw) {
      const int64_t row = r0 + c;
      unsigned long long okey = 0ull;
      bool match = true;
      if constexpr (FILTER)
        if (row < p.n) match = (p.mask[(size_t)(row >> 5) * p.mask_qs + qi] >> (row & 31)) & 1u;
      if (row < p.n && match) {
        okey = f64_orderable(exact_key_row<ST>(p.slot, (uint32_t)row, q, qn, lane));
        if (okey == 0ull) okey = 1ull;
      }
      if (lane == 0) {
        ek[kFbBest + c] = okey;
        ei[kFbBest + c] = row < p.n ? (uint32_t)row : 0xffffffffu;
        beat |= okey > kth;   // equal keys: the earlier row is already in the list and wins the tie
      }
    }
    if (beat) s_beats = 1;
    __syncthreads();
    if (s_beats) sort_exact_pairs(ek, ei, 2 * kFbBest, tid, nt);
    __syncthreads();
  }
  const RescoreArgs ra{p.slot, q, p.k, p.out_ids + (size_t)qi * p.k, p.out_scores + (size_t)qi * p.k, p.out_counts + qi};
  emit_exact_pairs(ek, ei, kFbBest, ra);
}

// ------------------------------------------------------------------------------------------------ filtered search
// Match mask of a chunk of <= 256 queries: bit (row % 32) of mask[(row / 32) * qs + q] is set iff row < n satisfies
// query q's program (sb_pred, DESIGN.md K1h; an empty program matches every row).  Legacy conjunctions and grouped
// search's exclusion mode arrive here as programs too (dense_topk_filtered_enqueue).  One launch serves a group of the
// chunk's DISTINCT programs, staged in shared memory with their code pools: each warp owns 32-row words (lane = row),
// loads each column the chunk references once per row into its own shared-memory slot, evaluates every distinct program
// once (boolean stack in a 64-bit register), ballots it, and writes the word to every query column that shares the
// program, so a block of 32 query columns is one 128-byte store.  counts[q] += popcount of its words.
constexpr int kGatherMax = 2048;   // queries with at most this many matching rows skip the scans (= winner buffer)
constexpr int kWhereThreads = 256;
constexpr int kWhereWarps = kWhereThreads / 32;
constexpr int kWhereMaxPreds = 1536;          // program steps of one launch (staged: 60 KB)
constexpr int kWhereMaxPoolStaged = 8192;     // codes of one launch's pools staged in shared memory; beyond: read from L2

struct WhereParams {
  const int32_t* tag[SB_MAX_TAG_FIELDS];      // the columns the chunk references; program fields index these
  const double* val[SB_MAX_VALUE_FIELDS];
  int32_t n_tag, n_val;
  const sb_pred* prog;                        // the launch's distinct programs, back to back
  const int32_t* u_off;                       // [n_u + 1] program u is prog[u_off[u], u_off[u+1])
  const int32_t* q_u;                         // [qs] query column -> program; -1 = zero column, -2 = another launch's
  const int32_t* pool;                        // IN codes (offsets relative to this pointer)
  int32_t n_preds, n_u, n_pool, pool_staged;
  int64_t n, n_words;
  int32_t qs;
  uint32_t* mask;                             // [n_words][qs]
  int32_t* counts;                            // [qs], zeroed by the caller
};

// true iff v is one of the n ascending codes at a (shared or global memory)
__device__ __forceinline__ bool sorted_codes_contain(const int32_t* a, int n, int32_t v) {
  int lo = 0, len = n;
  while (len > 0) {
    const int h = len >> 1;
    if (a[lo + h] < v) {
      lo += h + 1;
      len -= h + 1;
    } else {
      len = h;
    }
  }
  return lo < n && a[lo] == v;
}

// One program on this thread's row: tg / vl point at the thread's slot of column 0 (column c is c * kWhereThreads on).
// Bit 0 of st is the top of the stack; validation guarantees depth <= 64, so no bit is ever shifted out.
__device__ __forceinline__ bool where_eval(const sb_pred* pr, int len, const int32_t* pool, const int32_t* tg,
                                           const double* vl) {
  uint64_t st = 0ull;
  for (int i = 0; i < len; ++i) {
    const sb_pred& p = pr[i];
    const int op = p.op;
    bool r;
    if (op >= SB_PRED_AND) {
      const int na = p.a;
      const uint64_t m = na >= 64 ? ~0ull : (1ull << na) - 1ull;
      const uint64_t x = st & m;
      r = op == SB_PRED_AND ? x == m : op == SB_PRED_OR ? x != 0ull : op == SB_PRED_NOR ? x == 0ull : __popcll(x) >= p.b;
      st = na >= 64 ? 0ull : st >> na;
    } else if (op == SB_PRED_RANGE) {
      const double v = vl[p.field * kWhereThreads];
      r = (p.lo_incl ? v >= p.lo : v > p.lo) && (p.hi_incl ? v <= p.hi : v < p.hi);   // NaN: false
    } else {
      const int32_t t = tg[p.field * kWhereThreads];
      r = op == SB_PRED_EQ ? t == p.a : op == SB_PRED_PRESENT ? t >= 0 : sorted_codes_contain(pool + p.a, p.b, t);
    }
    st = (st << 1) | (r ? 1ull : 0ull);
  }
  return len == 0 || (st & 1ull) != 0ull;
}

// dynamic shared memory of one launch: values [n_val][256] | programs | tags [n_tag][256] | u_off | bits [8][n_u] | pool
__host__ __device__ inline size_t where_smem_bytes(int n_val, int n_preds, int n_tag, int n_u, int n_pool_staged) {
  return (size_t)n_val * kWhereThreads * 8 + (size_t)n_preds * sizeof(sb_pred) + (size_t)n_tag * kWhereThreads * 4 +
         (size_t)(n_u + 1) * 4 + (size_t)kWhereWarps * n_u * 4 + (size_t)n_pool_staged * 4;
}

__global__ void __launch_bounds__(kWhereThreads) dense_where_mask_kernel(const WhereParams p) {
  extern __shared__ __align__(16) uint8_t wsm[];
  double* s_val = reinterpret_cast<double*>(wsm);
  sb_pred* s_prog = reinterpret_cast<sb_pred*>(s_val + (size_t)p.n_val * kWhereThreads);
  int32_t* s_tag = reinterpret_cast<int32_t*>(s_prog + p.n_preds);
  int32_t* s_uoff = s_tag + (size_t)p.n_tag * kWhereThreads;
  uint32_t* s_bits = reinterpret_cast<uint32_t*>(s_uoff + p.n_u + 1);
  int32_t* s_pool = reinterpret_cast<int32_t*>(s_bits + kWhereWarps * p.n_u);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(p.prog);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(s_prog);
    const int words = p.n_preds * (int)(sizeof(sb_pred) / 8);
    for (int i = tid; i < words; i += kWhereThreads) dst[i] = __ldg(src + i);
    for (int i = tid; i <= p.n_u; i += kWhereThreads) s_uoff[i] = __ldg(p.u_off + i);
    if (p.pool_staged)
      for (int i = tid; i < p.n_pool; i += kWhereThreads) s_pool[i] = __ldg(p.pool + i);
  }
  __syncthreads();
  const int32_t* pool = p.pool_staged ? s_pool : p.pool;
  int qu[8], cnt[8];
#pragma unroll
  for (int qb = 0; qb < 8; ++qb) {
    qu[qb] = qb * 32 < p.qs ? __ldg(p.q_u + qb * 32 + lane) : -2;
    cnt[qb] = 0;
  }
  uint32_t* bits = s_bits + warp * p.n_u;
  int32_t* my_tag = s_tag + tid;
  double* my_val = s_val + tid;
  const int64_t warp0 = ((int64_t)blockIdx.x * kWhereThreads + tid) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * kWhereThreads) >> 5;
  for (int64_t w = warp0; w < p.n_words; w += nwarps) {
    const int64_t row = w * 32 + lane;
    const bool live = row < p.n;
    // each thread reads back only its own slots: no barrier between these stores and where_eval's loads
    for (int c = 0; c < p.n_tag; ++c) my_tag[c * kWhereThreads] = live ? __ldg(p.tag[c] + row) : -1;
    for (int c = 0; c < p.n_val; ++c) my_val[c * kWhereThreads] = live ? __ldg(p.val[c] + row) : __longlong_as_double(-1ll);
    for (int u = 0; u < p.n_u; ++u) {
      const int b0 = s_uoff[u];
      const bool m = live && where_eval(s_prog + b0, s_uoff[u + 1] - b0, pool, my_tag, my_val);
      const uint32_t b = __ballot_sync(0xffffffffu, m);
      if (lane == 0) bits[u] = b;
    }
    __syncwarp();
#pragma unroll
    for (int qb = 0; qb < 8; ++qb) {
      if (qu[qb] == -2) continue;
      const uint32_t mine = qu[qb] >= 0 ? bits[qu[qb]] : 0u;
      p.mask[(size_t)w * p.qs + qb * 32 + lane] = mine;
      cnt[qb] += __popc(mine);
    }
    __syncwarp();   // bits[] is rewritten for the next word
  }
#pragma unroll
  for (int qb = 0; qb < 8; ++qb)
    if (qu[qb] >= 0 && cnt[qb] > 0) atomicAdd(p.counts + qb * 32 + lane, cnt[qb]);
}

// Exact path of a low-cardinality query (<= kGatherMax matching rows): one CTA compacts the query's matching rows out
// of the mask and re-scores all of them in fp64 (rescore_and_emit, the same stage the scans end with).
struct GatherParams {
  const uint32_t* mask;
  int32_t qs;
  int64_t n_words;
  const int32_t* qlist;      // [grid] chunk-local query index of each CTA
  SlotView slot;
  const float* q;            // [nq][d_pad] the caller's fp32 queries
  int32_t k;
  int64_t* out_ids;
  double* out_scores;
  int32_t* out_counts;
};

template <int ST>
__global__ void __launch_bounds__(kMergeThreads, 1) dense_filter_gather_kernel(const GatherParams p) {
  extern __shared__ __align__(16) uint8_t gsmem[];
  unsigned long long* sel = reinterpret_cast<unsigned long long*>(gsmem);   // [kGatherMax] (key score field unused)
  unsigned long long* ek = sel + kGatherMax;                               // [kGatherMax]
  uint32_t* ei = reinterpret_cast<uint32_t*>(ek + kGatherMax);             // [kGatherMax]
  float* q_s = reinterpret_cast<float*>(ei + kGatherMax);                  // [d_pad]
  __shared__ double qq_s;
  __shared__ int s_n;
  const int qi = p.qlist[blockIdx.x];
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  for (int64_t w = threadIdx.x; w < p.n_words; w += blockDim.x) {
    uint32_t bits = p.mask[(size_t)w * p.qs + qi];
    if (bits == 0u) continue;
    int at = atomicAdd(&s_n, __popc(bits));
    for (; bits != 0u; bits &= bits - 1u, ++at)
      if (at < kGatherMax) sel[at] = make_key32(0.f, (uint32_t)(w * 32 + __ffs(bits) - 1));
  }
  __syncthreads();
  const int nsel = min(s_n, kGatherMax);   // the host routes only queries with <= kGatherMax matches here
  int P = 32;
  while (P < nsel) P <<= 1;
  const RescoreArgs ra{p.slot, p.q + (size_t)qi * p.slot.d_pad, p.k, p.out_ids + (size_t)qi * p.k,
                       p.out_scores + (size_t)qi * p.k, p.out_counts + qi};
  rescore_and_emit<ST>(sel, nsel, P, ek, ei, &qq_s, q_s, ra);
}

// ------------------------------------------------------------------------------------------------ grouped search (K1f)
constexpr int kGroupThreads = 1024;   // >= the longest round prefix (kDenseMaxK)

struct GroupCollectParams {
  const int64_t* ids;       // [nq][K] one round's exact prefix, best first (id_base + row)
  const double* scores;     // [nq][K]
  const int32_t* counts;    // [nq] prefix length (= K: the prefix is full)
  const int32_t* qmap;      // [nq] grouped query of each round query; nullptr = the identity
  const int32_t* tag;       // the group_by tag column
  int64_t id_base;
  int32_t K, L, G;
  int32_t* n_groups;        // [B] groups found so far
  int32_t* g_code;          // [B][L] group codes, in order of their best row
  int32_t* g_hits;          // [B][L] hits recorded per group (<= G)
  int64_t* h_ids;           // [B][L][G]
  double* h_scores;         // [B][L][G]
};

// One CTA per round query; thread t owns prefix position t.  Sorting the (code, position) pairs gives every position its
// rank inside its group, its group's first position and the group's count in the prefix; an exclusive scan over "first
// position of its group" numbers the groups in the order of their best row.  A round's groups are all new (an exclusion
// round excludes the groups found before it), so they are numbered on from n_groups.  A position is recorded iff its
// group number is < L and its rank < G.
__global__ void __launch_bounds__(kGroupThreads) dense_group_collect_kernel(const GroupCollectParams p) {
  __shared__ unsigned long long key[kGroupThreads];
  __shared__ int rank_of[kGroupThreads], first_of[kGroupThreads], run_of[kGroupThreads], ord[kGroupThreads];
  __shared__ int warp_sum[kGroupThreads / 32];
  const int qi = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int b = p.qmap ? p.qmap[qi] : qi;
  const int cnt = p.counts[qi];
  const int base = p.n_groups[b];
  const int64_t* ids = p.ids + (size_t)qi * p.K;
  int32_t code = -1;
  if (t < cnt) code = __ldg(p.tag + (ids[t] - p.id_base));
  // (code, position) ascending, rows without a group last: sorted descending as complements (0 = no group)
  key[t] = code >= 0 ? ~(((unsigned long long)(uint32_t)code << 32) | (uint32_t)t) : 0ull;
  rank_of[t] = -1;
  __syncthreads();
  int P = 32;
  while (P < cnt) P <<= 1;
  block_sort_desc_u64(key, P, t, kGroupThreads);
  if (t < P && key[t] != 0ull) {
    const uint32_t c = (uint32_t)(~key[t] >> 32);
    int lo = 0, hi = t;   // first sorted position of code c
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if ((uint32_t)(~key[m] >> 32) < c) lo = m + 1;
      else hi = m;
    }
    int lo2 = t + 1, hi2 = P;   // first sorted position past code c (a complemented 0 reads as code 0xffffffff)
    while (lo2 < hi2) {
      const int m = (lo2 + hi2) >> 1;
      if ((uint32_t)(~key[m] >> 32) <= c) lo2 = m + 1;
      else hi2 = m;
    }
    const int pos = (int)(uint32_t)~key[t];
    rank_of[pos] = t - lo;
    first_of[pos] = (int)(uint32_t)~key[lo];
    run_of[pos] = lo2 - lo;
  }
  __syncthreads();
  const int flag = (t < cnt && rank_of[t] == 0) ? 1 : 0;
  int incl = flag;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_sum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int v = warp_sum[lane];
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += y;
    }
    warp_sum[lane] = v;
  }
  __syncthreads();
  ord[t] = incl - flag + (warp ? warp_sum[warp - 1] : 0);
  __syncthreads();
  if (t < cnt && rank_of[t] >= 0) {
    const int g = base + ord[first_of[t]];
    const int r = rank_of[t];
    if (g < p.L && r < p.G) {
      const size_t h = ((size_t)b * p.L + g) * p.G + r;
      p.h_ids[h] = ids[t];
      p.h_scores[h] = p.scores[(size_t)qi * p.K + t];
      if (r == 0) {
        p.g_code[(size_t)b * p.L + g] = code;
        p.g_hits[(size_t)b * p.L + g] = min(run_of[t], p.G);
      }
    }
  }
  if (t == 0) p.n_groups[b] = min(p.L, base + warp_sum[31]);
}

// out[r] = q_pad[src[r]]: one operand row per round query or completion pair
__global__ void __launch_bounds__(256) dense_group_queries_kernel(const float* __restrict__ q_pad,
                                                                  const int32_t* __restrict__ src, int d_pad,
                                                                  float* __restrict__ out) {
  const float* s = q_pad + (size_t)src[blockIdx.x] * d_pad;
  for (int i = threadIdx.x; i < d_pad; i += blockDim.x) out[(size_t)blockIdx.x * d_pad + i] = s[i];
}

// A completion's top-G of one group (filtered search, [np][G]) replaces that group's hits: pair i -> group dest[i]
struct GroupAssembleParams {
  const int64_t* ids;
  const double* scores;
  const int32_t* counts;
  const int32_t* dest;      // [np] b * L + g
  int32_t G;
  int64_t n;                // np * G
  int32_t* g_hits;
  int64_t* h_ids;
  double* h_scores;
};

__global__ void __launch_bounds__(256) dense_group_assemble_kernel(const GroupAssembleParams p) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  const int64_t pr = i / p.G, r = i % p.G;
  const int32_t g = p.dest[pr];
  p.h_ids[(size_t)g * p.G + r] = p.ids[i];
  p.h_scores[(size_t)g * p.G + r] = p.scores[i];
  if (r == 0) p.g_hits[g] = p.counts[pr];
}

// ------------------------------------------------------------------------------------------------ host side
constexpr int kDenseMaxK = 1024;  // per-call top_k limit of both scans (per-CTA lists / winner buffers)

int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

struct ScanPlan {
  int nchunk, rw, qb_max, kprime, bcap, stages, grid, num_tiles;
  uint32_t tile_bytes;
  size_t scan_smem, merge_smem;
  int heads_per_list, heads_pow2;
};

int supported_nchunk(int ch) {
  const int need = (ch + 31) / 32;
  static const int sup[] = {1, 2, 3, 4, 6, 8, 12, 16};
  for (int s : sup)
    if (s >= need) return s;
  return -1;
}

int make_plan(sb_ctx* ctx, const DenseIndex& ix, int k, ScanPlan* pl) {
  const int ch = ix.d_pad / 8;
  pl->nchunk = supported_nchunk(ch);
  SB_REQUIRE(pl->nchunk > 0, SB_ERR_UNSUPPORTED, "dense: dimension %d too large (max 4096)", ix.d);
  pl->rw = pl->nchunk <= 4 ? 4 : (pl->nchunk <= 8 ? 2 : 1);
  pl->qb_max = pl->nchunk <= 4 ? 4 : (pl->nchunk <= 8 ? 2 : 1);
  // per-CTA list length: >= k (the k-th best approximate key must be in the lists); the spare entries above k are what
  // usually lets a list serve the error window without a fallback
  pl->kprime = next_pow2(k + 28);
  if (pl->kprime < 128) pl->kprime = 128;
  if (pl->kprime > kDenseMaxK) pl->kprime = kDenseMaxK;
  SB_REQUIRE(k <= kDenseMaxK, SB_ERR_UNSUPPORTED, "dense: top_k %d too large (max %d per call)", k, kDenseMaxK);
  const int R = kConsumerWarps * pl->rw;
  // compaction sorts best[K'] + one batch in registers across one warp: 512 / 1024 / 1024 / 2048 keys
  pl->bcap = pl->kprime <= 256 ? 3 * pl->kprime : pl->kprime;
  pl->tile_bytes = (uint32_t)R * (uint32_t)ix.d_pad * 2u;
  pl->num_tiles = (int)(ix.n_pad / R);
  const size_t budget = ctx->smem_optin;
  const size_t per_q = (size_t)(pl->kprime + 2 * pl->bcap) * 8;
  const size_t scratch = (pl->kprime + pl->bcap == 512) ? 0 : (size_t)(pl->kprime + pl->bcap) * 8;
  while ((size_t)pl->qb_max * per_q + scratch + 1024 + 2 * (size_t)pl->tile_bytes > budget) {
    if (pl->qb_max > 1) { pl->qb_max >>= 1; continue; }
    sb_set_error("dense: configuration does not fit shared memory (d=%d, k=%d)", ix.d, k);
    return SB_ERR_UNSUPPORTED;
  }
  const size_t fixed = (size_t)pl->qb_max * per_q + scratch;
  int stages = (int)((budget - fixed - 1024) / pl->tile_bytes);
  if (stages > 8) stages = 8;
  if (stages < 2) stages = 2;
  pl->stages = stages;
  pl->scan_smem = (size_t)stages * pl->tile_bytes + fixed + 2 * 8 * (size_t)stages + 256;
  pl->grid = ctx->num_sms < pl->num_tiles ? ctx->num_sms : pl->num_tiles;
  if (pl->grid < 1) pl->grid = 1;
  pl->heads_per_list = (pl->kprime + pl->grid - 1) / pl->grid;
  pl->heads_pow2 = next_pow2(pl->grid * pl->heads_per_list);
  SB_REQUIRE(pl->heads_pow2 <= kSelCap, SB_ERR_UNSUPPORTED, "dense: internal merge capacity exceeded");
  pl->merge_smem = (size_t)kSelCap * 20 + (size_t)ix.d_pad * 4 + 64;
  return SB_OK;
}

template <int NCHUNK, int QB, int RW, bool FILTER, bool EUCLID>
int launch_scan(const ScanParams& sp, const ScanPlan& pl, cudaStream_t st) {
  if (sp.ch == NCHUNK * 32) {
    auto kern = dense_scan_kernel<NCHUNK, QB, RW, true, FILTER, EUCLID>;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.scan_smem));
    kern<<<pl.grid, kScanThreads, pl.scan_smem, st>>>(sp);
  } else {
    auto kern = dense_scan_kernel<NCHUNK, QB, RW, false, FILTER, EUCLID>;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.scan_smem));
    kern<<<pl.grid, kScanThreads, pl.scan_smem, st>>>(sp);
  }
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

template <int NCHUNK, int RW, bool FILTER, bool EUCLID>
int dispatch_qb(int qb, const ScanParams& sp, const ScanPlan& pl, cudaStream_t st) {
  if constexpr (NCHUNK <= 4) {
    if (qb == 4) return launch_scan<NCHUNK, 4, RW, FILTER, EUCLID>(sp, pl, st);
  }
  if constexpr (NCHUNK <= 8) {
    if (qb == 2) return launch_scan<NCHUNK, 2, RW, FILTER, EUCLID>(sp, pl, st);
  }
  return launch_scan<NCHUNK, 1, RW, FILTER, EUCLID>(sp, pl, st);
}

template <bool FILTER, bool EUCLID>
int dispatch_scan(int qb, const ScanParams& sp, const ScanPlan& pl, cudaStream_t st) {
  switch (pl.nchunk) {
    case 1: return dispatch_qb<1, 4, FILTER, EUCLID>(qb, sp, pl, st);
    case 2: return dispatch_qb<2, 4, FILTER, EUCLID>(qb, sp, pl, st);
    case 3: return dispatch_qb<3, 4, FILTER, EUCLID>(qb, sp, pl, st);
    case 4: return dispatch_qb<4, 4, FILTER, EUCLID>(qb, sp, pl, st);
    case 6: return dispatch_qb<6, 2, FILTER, EUCLID>(qb, sp, pl, st);
    case 8: return dispatch_qb<8, 2, FILTER, EUCLID>(qb, sp, pl, st);
    case 12: return dispatch_qb<12, 1, FILTER, EUCLID>(qb, sp, pl, st);
    case 16: return dispatch_qb<16, 1, FILTER, EUCLID>(qb, sp, pl, st);
  }
  sb_set_error("dense: unsupported chunk count %d", pl.nchunk);
  return SB_ERR_UNSUPPORTED;
}

// Cosine and Dot run the same (acc * scale) kernels; Euclid its own instantiations
int dispatch_scan_metric(int metric, bool filter, int qb, const ScanParams& sp, const ScanPlan& pl, cudaStream_t st) {
  if (metric == SB_METRIC_EUCLID)
    return filter ? dispatch_scan<true, true>(qb, sp, pl, st) : dispatch_scan<false, true>(qb, sp, pl, st);
  return filter ? dispatch_scan<true, false>(qb, sp, pl, st) : dispatch_scan<false, false>(qb, sp, pl, st);
}

// q_pad: [B][d_pad] fp32 device, zero padded.  Enqueues all scan passes of a chunk of queries, then ONE merge launch
// (one CTA per query) for the whole chunk.
constexpr int kMergeChunk = 256;

int dense_topk_enqueue(sb_ctx* ctx, DenseIndex& ix, const float* q_pad, int B, int k, int64_t* out_ids,
                       double* out_scores, int32_t* out_counts, cudaStream_t st, const DenseFilter* flt = nullptr) {
  ScanPlan pl;
  int rc = make_plan(ctx, ix, k, &pl);
  if (rc) return rc;
  // batches of >= 16 queries ride the tensor cores: one HBM pass per 64 / 128 queries instead of one per 4.  A uint8 slot
  // has no fp16 rows for the CUDA-core scan: every batch takes the wgmma scan (DESIGN.md K1i)
  if (ix.storage == SB_STORAGE_U8 || (ctx->dense_mode != 1 && dense_mma_eligible(ctx, ix, B)))
    return dense_mma_topk_enqueue(ctx, ix, q_pad, B, k, out_ids, out_scores, out_counts, st, flt);
  const int chunk = B < kMergeChunk ? B : kMergeChunk;
  const size_t per_q = (size_t)pl.grid * pl.kprime;
  rc = ctx->cand_dev.reserve((size_t)chunk * per_q * 8);
  if (rc) return rc;
  // normalised queries for the scan, eps + fallback flags for the hand-off
  float *qn = nullptr, *eps = nullptr, *rq = nullptr;
  int32_t* fb = nullptr;
  if ((rc = dense_prep_queries(ctx, ix, q_pad, B, B, /*mma=*/false, &qn, nullptr, &eps, &fb, &rq, st))) return rc;
  const bool f32 = ix.storage == SB_STORAGE_F32;
  auto merge_kern = flt ? (f32 ? dense_merge_kernel<true, true> : dense_merge_kernel<true, false>)
                        : (f32 ? dense_merge_kernel<false, true> : dense_merge_kernel<false, false>);
  SB_CUDA(cudaFuncSetAttribute(merge_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.merge_smem));
  for (int c0 = 0; c0 < B; c0 += chunk) {
    const int nq = std::min(chunk, B - c0);
    int b0 = 0;
    while (b0 < nq) {
      int qb = pl.qb_max;
      while (qb > nq - b0) qb >>= 1;
      if (flt) {   // a pass whose queries are all answered by the gather path is not launched
        bool any = false;
        for (int i = 0; i < qb; ++i) any |= flt->state_host[c0 + b0 + i] == 0;
        if (!any) {
          b0 += qb;
          continue;
        }
      }
      ScanParams sp;
      sp.rows = ix.rows;
      sp.inv_norm = ix.inv_norm;
      sp.q = qn + (size_t)(c0 + b0) * ix.d_pad;
      sp.cand = ctx->cand_dev.as<unsigned long long>() + (size_t)b0 * per_q;
      sp.n = ix.n;
      sp.d_pad = ix.d_pad;
      sp.ch = ix.d_pad / 8;
      sp.num_tiles = pl.num_tiles;
      sp.kprime = pl.kprime;
      sp.bcap = pl.bcap;
      sp.stages = pl.stages;
      sp.tile_bytes = pl.tile_bytes;
      sp.mask = flt ? flt->mask + (c0 + b0) : nullptr;
      sp.mask_qs = flt ? flt->qs : 0;
      sp.state = flt ? flt->state + (c0 + b0) : nullptr;
      sp.hh = ix.hh;
      sp.rq = rq ? rq + (c0 + b0) : nullptr;
      {
        ProfScope ps(ctx, SB_PROF_DENSE_SCAN, st);
        rc = dispatch_scan_metric(ix.metric, flt != nullptr, qb, sp, pl, st);
      }
      if (rc) return rc;
      b0 += qb;
    }
    MergeParams mp;
    mp.cand = ctx->cand_dev.as<unsigned long long>();
    mp.G = pl.grid;
    mp.kprime = pl.kprime;
    mp.heads_per_list = pl.heads_per_list;
    mp.heads_pow2 = pl.heads_pow2;
    mp.slot = slot_view(ix);
    mp.q = q_pad + (size_t)c0 * ix.d_pad;
    mp.eps = eps + c0;
    mp.fallback = fb + c0;
    mp.k = k;
    mp.out_ids = out_ids + (size_t)c0 * k;
    mp.out_scores = out_scores + (size_t)c0 * k;
    mp.out_counts = out_counts + c0;
    mp.state = flt ? flt->state + c0 : nullptr;
    {
      ProfScope ps(ctx, SB_PROF_DENSE_MERGE, st);
      merge_kern<<<nq, kMergeThreads, pl.merge_smem, st>>>(mp);
    }
    SB_CUDA(cudaGetLastError());
  }
  return dense_fallback_enqueue(ctx, ix, q_pad, B, k, fb, out_ids, out_scores, out_counts, st, flt);
}

__global__ void fill_empty_topk_kernel(int64_t* ids, double* sc, int32_t* cnt, int B, int k) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * k) {
    ids[i] = -1;
    sc[i] = 0.0;
  }
  if (i < B) cnt[i] = 0;
}

// the stored vector: y (Cosine), c * y in fp64 rounded to fp32 (Dot / Euclid, cfac != nullptr)
__global__ void dense_fetch_kernel(const __half* rows, const double* cfac, int d, int d_pad, int64_t n, int64_t id_base,
                                   const int64_t* ids, int n_ids, float* out) {
  int r = blockIdx.x;
  if (r >= n_ids) return;
  int64_t idx = ids[r] - id_base;
  const bool live = idx >= 0 && idx < n;
  const double c = (cfac && live) ? cfac[idx] : 1.0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    float v = 0.f;
    if (live) v = cfac ? (float)(c * (double)__half2float(rows[(size_t)idx * d_pad + i]))
                       : __half2float(rows[(size_t)idx * d_pad + i]);
    out[(size_t)r * d + i] = v;
  }
}

// float32 storage: x bit for bit; normalise = Cosine: fl32(x / ||x||) with ||x|| in fp64 (a zero row stays zero)
__global__ void __launch_bounds__(128) dense_fetch_f32_kernel(const float* rows32, bool normalise, int d, int d_pad,
                                                              int64_t n, int64_t id_base, const int64_t* ids, int n_ids,
                                                              float* out) {
  __shared__ double s_red[4];
  const int r = blockIdx.x;
  if (r >= n_ids) return;
  const int64_t idx = ids[r] - id_base;
  const bool live = idx >= 0 && idx < n;
  const float* x = rows32 + (size_t)(live ? idx : 0) * d_pad;
  double nrm = 1.0;
  if (normalise) {
    double ss = 0.0;
    if (live)
      for (int i = threadIdx.x; i < d; i += blockDim.x) ss = __fma_rn((double)x[i], (double)x[i], ss);
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = ss;
    __syncthreads();
    const double t = s_red[0] + s_red[1] + s_red[2] + s_red[3];
    nrm = t > 0.0 ? sqrt(t) : 1.0;
  }
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    float v = 0.f;
    if (live) v = normalise ? (float)((double)x[i] / nrm) : x[i];
    out[(size_t)r * d + i] = v;
  }
}

// uint8 storage: x as fp32 for every metric (a normalised uint8 vector does not exist)
__global__ void __launch_bounds__(128) dense_fetch_u8_kernel(const uint8_t* rows8, int d, int d_pad, int64_t n,
                                                             int64_t id_base, const int64_t* ids, int n_ids, float* out) {
  const int r = blockIdx.x;
  if (r >= n_ids) return;
  const int64_t idx = ids[r] - id_base;
  const bool live = idx >= 0 && idx < n;
  for (int i = threadIdx.x; i < d; i += blockDim.x) out[(size_t)r * d + i] = live ? (float)rows8[(size_t)idx * d_pad + i] : 0.f;
}

}  // namespace

// Shared with dense_mma.cu: query preparation (normalised fp32 copy, optional fp16 operand rows, eps, cleared fallback
// flags) and the brute-force fallback launch.  `rows` >= B operand rows are prepared (rows >= B are zero padding).
int dense_prep_queries(sb_ctx* ctx, const DenseIndex& ix, const float* q_pad, int B, int rows, bool mma, float** qn_out,
                       __half* q16, float** eps_out, int32_t** fb_out, float** rq_out, cudaStream_t st) {
  int rc;
  if ((rc = ctx->qaux_dev.reserve((size_t)rows * 12 + 64))) return rc;
  float* eps = ctx->qaux_dev.as<float>();
  int32_t* fb = reinterpret_cast<int32_t*>(eps + rows);
  PrepMetric pm;
  pm.metric = ix.metric;
  pm.rho = ix.rho_max;
  pm.hmax = ix.h_max;
  pm.sigma = ix.sigma_max;
  pm.rq =ix.metric == SB_METRIC_EUCLID ? reinterpret_cast<float*>(fb + rows) : nullptr;
  pm.fb = fb;
  *rq_out = pm.rq;
  float* qn = nullptr;
  if (qn_out) {
    if ((rc = ctx->qn_dev.reserve((size_t)rows * ix.d_pad * sizeof(float)))) return rc;
    qn = ctx->qn_dev.as<float>();
    *qn_out = qn;
  }
  SB_CUDA(cudaMemsetAsync(fb, 0, (size_t)rows * 4, st));
  ctx->launches += 1;
  if (ix.storage == SB_STORAGE_U8)
    dense_prep_queries_kernel<SB_STORAGE_U8><<<rows, 256, 0, st>>>(q_pad, B, ix.d_pad, qn, q16, eps, mma ? 1 : 0, pm);
  else if (ix.storage == SB_STORAGE_F32)
    dense_prep_queries_kernel<SB_STORAGE_F32><<<rows, 256, 0, st>>>(q_pad, B, ix.d_pad, qn, q16, eps, mma ? 1 : 0, pm);
  else
    dense_prep_queries_kernel<SB_STORAGE_F16><<<rows, 256, 0, st>>>(q_pad, B, ix.d_pad, qn, q16, eps, mma ? 1 : 0, pm);
  SB_CUDA(cudaGetLastError());
  *eps_out = eps;
  *fb_out = fb;
  return SB_OK;
}

int dense_fallback_enqueue(sb_ctx* ctx, const DenseIndex& ix, const float* q_pad, int B, int k, const int32_t* fb,
                           int64_t* out_ids, double* out_scores, int32_t* out_counts, cudaStream_t st,
                           const DenseFilter* flt) {
  if (ctx->fb_count_dev.cap == 0) {
    int rc = ctx->fb_count_dev.reserve(8);
    if (rc) return rc;
    SB_CUDA(cudaMemsetAsync(ctx->fb_count_dev.p, 0, 8, st));
  }
  FallbackParams fp;
  fp.counter = ctx->fb_count_dev.as<unsigned long long>();
  fp.mask = flt ? flt->mask : nullptr;
  fp.mask_qs = flt ? flt->qs : 0;
  fp.flag = fb;
  fp.slot = slot_view(ix);
  fp.q = q_pad;
  fp.n = ix.n;
  fp.k = k;
  fp.out_ids = out_ids;
  fp.out_scores = out_scores;
  fp.out_counts = out_counts;
  ctx->launches += 1;
  auto kern = flt ? dense_exact_fallback_kernel<true, SB_STORAGE_F16> : dense_exact_fallback_kernel<false, SB_STORAGE_F16>;
  if (ix.storage == SB_STORAGE_F32)
    kern = flt ? dense_exact_fallback_kernel<true, SB_STORAGE_F32> : dense_exact_fallback_kernel<false, SB_STORAGE_F32>;
  else if (ix.storage == SB_STORAGE_U8)
    kern = flt ? dense_exact_fallback_kernel<true, SB_STORAGE_U8> : dense_exact_fallback_kernel<false, SB_STORAGE_U8>;
  kern<<<B, kFbThreads, 0, st>>>(fp);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

namespace {

size_t align16(size_t v) { return (v + 15) / 16 * 16; }

// The public program input, checked before anything is launched: offsets, op codes, loaded fields, pool ranges in bounds
// and ascending, a well-formed stack, the limits (include/sentio_b200.h, sb_dense_topk_where).
int where_validate(const char* who, const DenseIndex& ix, int B, const int32_t* p_off, const sb_pred* prog,
                   const int32_t* pool, int32_t n_pool) {
  SB_REQUIRE(p_off[0] == 0, SB_ERR_ARG, "%s: p_off[0] must be 0", who);
  SB_REQUIRE(n_pool >= 0 && (n_pool == 0 || pool != nullptr), SB_ERR_ARG, "%s: bad pool (n_pool=%d)", who, n_pool);
  for (int b = 0; b < B; ++b) {
    const int32_t p0 = p_off[b], p1 = p_off[b + 1];
    SB_REQUIRE(p1 >= p0, SB_ERR_ARG, "%s: p_off is not non-decreasing at %d", who, b);
    SB_REQUIRE(p1 - p0 <= SB_MAX_PRED, SB_ERR_ARG, "%s: query %d has %d program steps (max %d)", who, b, p1 - p0,
               SB_MAX_PRED);
    int depth = 0;
    for (int32_t i = p0; i < p1; ++i) {
      const sb_pred& e = prog[i];
      SB_REQUIRE(e.op >= SB_PRED_EQ && e.op <= SB_PRED_ATLEAST, SB_ERR_ARG, "%s: step %d has op %d", who, i, e.op);
      if (e.op == SB_PRED_RANGE) {
        SB_REQUIRE(e.field >= 0 && e.field < SB_MAX_VALUE_FIELDS, SB_ERR_ARG, "%s: step %d: value field %d out of range",
                   who, i, e.field);
        SB_REQUIRE(ix.vals[e.field] != nullptr, SB_ERR_STATE, "%s: value field %d has no column loaded", who, e.field);
        SB_REQUIRE(!std::isnan(e.lo) && !std::isnan(e.hi), SB_ERR_ARG, "%s: step %d: NaN range bound", who, i);
        SB_REQUIRE((e.lo_incl == 0 || e.lo_incl == 1) && (e.hi_incl == 0 || e.hi_incl == 1), SB_ERR_ARG,
                   "%s: step %d: inclusive flags must be 0 or 1", who, i);
      } else if (e.op <= SB_PRED_PRESENT) {
        SB_REQUIRE(e.field >= 0 && e.field < SB_MAX_TAG_FIELDS, SB_ERR_ARG, "%s: step %d: tag field %d out of range", who,
                   i, e.field);
        SB_REQUIRE(ix.tags[e.field] != nullptr, SB_ERR_STATE, "%s: field %d has no tag column loaded", who, e.field);
        SB_REQUIRE(e.op != SB_PRED_EQ || e.a >= 0, SB_ERR_ARG, "%s: step %d: EQ code %d (must be >= 0)", who, i, e.a);
        if (e.op == SB_PRED_IN) {
          SB_REQUIRE(e.a >= 0 && e.b >= 0 && (int64_t)e.a + e.b <= n_pool, SB_ERR_ARG,
                     "%s: step %d: pool range [%d, %d + %d) outside [0, %d)", who, i, e.a, e.a, e.b, n_pool);
          for (int32_t j = e.a; j < e.a + e.b; ++j)
            SB_REQUIRE(pool[j] >= 0 && (j == e.a || pool[j] > pool[j - 1]), SB_ERR_ARG,
                       "%s: step %d: pool codes must be >= 0 and strictly ascending (pool[%d] = %d)", who, i, j, pool[j]);
        }
      }
      if (e.op <= SB_PRED_PRESENT) {
        depth += 1;
      } else {
        SB_REQUIRE(e.a >= 0 && e.a <= depth, SB_ERR_ARG, "%s: step %d pops %d of %d stack entries", who, i, e.a, depth);
        depth += 1 - e.a;
      }
      SB_REQUIRE(depth <= SB_MAX_PRED_STACK, SB_ERR_ARG, "%s: query %d's program needs more than %d stack entries", who,
                 b, SB_MAX_PRED_STACK);
    }
    SB_REQUIRE(p1 == p0 || depth == 1, SB_ERR_ARG, "%s: query %d's program leaves %d stack entries (must be 1)", who, b,
               depth);
  }
  return SB_OK;
}

// One mask launch of a chunk: a group of its distinct programs (staged at the given offsets of the chunk's bytes)
struct WhereLaunch {
  size_t o_prog, o_uoff, o_qu, o_pool;
  int n_preds, n_u, n_pool;
};

// The host side of one chunk's mask: its distinct programs in launch groups, fields remapped to the chunk's columns
struct WhereChunk {
  std::vector<uint8_t> bytes;
  std::vector<WhereLaunch> launches;
  int n_tag = 0, n_val = 0;
  int tag_f[SB_MAX_TAG_FIELDS], val_f[SB_MAX_VALUE_FIELDS];
};

template <typename T>
size_t put(std::vector<uint8_t>& v, const T* src, size_t n) {
  const size_t o = (v.size() + 15) / 16 * 16;
  v.resize(o + n * sizeof(T));
  if (n) memcpy(v.data() + o, src, n * sizeof(T));
  return o;
}

void where_plan_chunk(const int32_t* p_off, const sb_pred* prog, const int32_t* pool, int c0, int nq, int qs,
                      WhereChunk& ch) {
  int slot_t[SB_MAX_TAG_FIELDS], slot_v[SB_MAX_VALUE_FIELDS];
  std::fill(slot_t, slot_t + SB_MAX_TAG_FIELDS, -1);
  std::fill(slot_v, slot_v + SB_MAX_VALUE_FIELDS, -1);
  // distinct programs by content (an IN leaf by its codes, not by where they sit in the pool)
  std::unordered_map<std::string, int> seen;
  std::vector<int> uq(nq), rep;
  for (int q = 0; q < nq; ++q) {
    std::string key;
    for (int32_t i = p_off[c0 + q]; i < p_off[c0 + q + 1]; ++i) {
      const sb_pred& e = prog[i];
      key.append(reinterpret_cast<const char*>(&e.op), 8);   // op, field
      if (e.op == SB_PRED_IN) {
        key.append(reinterpret_cast<const char*>(&e.b), 4);
        key.append(reinterpret_cast<const char*>(pool + e.a), (size_t)e.b * 4);
      } else {
        key.append(reinterpret_cast<const char*>(&e.a), sizeof(sb_pred) - 8);
      }
    }
    auto it = seen.emplace(key, (int)rep.size());
    if (it.second) rep.push_back(q);
    uq[q] = it.first->second;
  }
  // launch groups of consecutive distinct programs, each within the staged-program budget (SB_MAX_PRED <= the budget)
  std::vector<int> group_of(rep.size()), local(rep.size());
  std::vector<int> g_first;
  int cur = 0;
  for (size_t u = 0; u < rep.size(); ++u) {
    const int len = p_off[c0 + rep[u] + 1] - p_off[c0 + rep[u]];
    if (g_first.empty() || cur + len > kWhereMaxPreds) {
      g_first.push_back((int)u);
      cur = 0;
    }
    group_of[u] = (int)g_first.size() - 1;
    local[u] = (int)u - g_first.back();
    cur += len;
  }
  for (size_t g = 0; g < g_first.size(); ++g) {
    const size_t u1 = g + 1 < g_first.size() ? (size_t)g_first[g + 1] : rep.size();
    std::vector<sb_pred> gp;
    std::vector<int32_t> uoff(1, 0), gpool, qu(qs);
    for (size_t u = g_first[g]; u < u1; ++u) {
      const int q = rep[u];
      for (int32_t i = p_off[c0 + q]; i < p_off[c0 + q + 1]; ++i) {
        sb_pred e = prog[i];
        if (e.op == SB_PRED_RANGE) {
          if (slot_v[e.field] < 0) {
            slot_v[e.field] = ch.n_val;
            ch.val_f[ch.n_val++] = e.field;
          }
          e.field = slot_v[e.field];
        } else if (e.op <= SB_PRED_PRESENT) {
          if (slot_t[e.field] < 0) {
            slot_t[e.field] = ch.n_tag;
            ch.tag_f[ch.n_tag++] = e.field;
          }
          e.field = slot_t[e.field];
          if (e.op == SB_PRED_IN) {
            const int32_t a = (int32_t)gpool.size();
            gpool.insert(gpool.end(), pool + e.a, pool + e.a + e.b);
            e.a = a;
          }
        } else {
          e.field = 0;
        }
        gp.push_back(e);
      }
      uoff.push_back((int32_t)gp.size());
    }
    for (int q = 0; q < qs; ++q)
      qu[q] = q >= nq ? (g == 0 ? -1 : -2) : group_of[uq[q]] == (int)g ? local[uq[q]] : -2;
    WhereLaunch L;
    L.n_preds = (int)gp.size();
    L.n_u = (int)(u1 - g_first[g]);
    L.n_pool = (int)gpool.size();
    L.o_prog = put(ch.bytes, gp.data(), gp.size());
    L.o_uoff = put(ch.bytes, uoff.data(), uoff.size());
    L.o_qu = put(ch.bytes, qu.data(), qu.size());
    L.o_pool = put(ch.bytes, gpool.data(), gpool.size());
    ch.launches.push_back(L);
  }
}

// The mask launches of one planned chunk whose programs are staged on the device at sd (kernel attribute already set)
int where_mask_launches(sb_ctx* ctx, const DenseIndex& ix, const WhereChunk& ch, const uint8_t* sd, uint32_t* mask,
                        int32_t* cnt_d, int qs, cudaStream_t st) {
  const int64_t n_words = ix.n_pad / 32;
  WhereParams wp;
  for (int c = 0; c < ch.n_tag; ++c) wp.tag[c] = ix.tags[ch.tag_f[c]];
  for (int c = 0; c < ch.n_val; ++c) wp.val[c] = ix.vals[ch.val_f[c]];
  wp.n_tag = ch.n_tag;
  wp.n_val = ch.n_val;
  wp.n = ix.n;
  wp.n_words = n_words;
  wp.qs = qs;
  wp.mask = mask;
  wp.counts = cnt_d;
  for (const WhereLaunch& L : ch.launches) {
    wp.prog = reinterpret_cast<const sb_pred*>(sd + L.o_prog);
    wp.u_off = reinterpret_cast<const int32_t*>(sd + L.o_uoff);
    wp.q_u = reinterpret_cast<const int32_t*>(sd + L.o_qu);
    wp.pool = reinterpret_cast<const int32_t*>(sd + L.o_pool);
    wp.n_preds = L.n_preds;
    wp.n_u = L.n_u;
    wp.n_pool = L.n_pool;
    wp.pool_staged = L.n_pool <= kWhereMaxPoolStaged ? 1 : 0;
    const size_t smem = where_smem_bytes(ch.n_val, L.n_preds, ch.n_tag, L.n_u, wp.pool_staged ? L.n_pool : 0);
    const int64_t blocks = std::min<int64_t>((n_words + kWhereWarps - 1) / kWhereWarps, (int64_t)ctx->num_sms * 8);
    ProfScope ps(ctx, SB_PROF_DENSE_FILTER, st);
    dense_where_mask_kernel<<<(unsigned)blocks, kWhereThreads, smem, st>>>(wp);
  }
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

// largest dynamic shared memory of a planned chunk's mask launches
size_t where_chunk_smem(const WhereChunk& ch) {
  size_t m = 0;
  for (const WhereLaunch& L : ch.launches) {
    const int staged = L.n_pool <= kWhereMaxPoolStaged ? L.n_pool : 0;
    m = std::max(m, where_smem_bytes(ch.n_val, L.n_preds, ch.n_tag, L.n_u, staged));
  }
  return m;
}

}  // namespace

int dense_where_mask(sb_ctx* ctx, DenseIndex& ix, const int32_t* p_off, const sb_pred* prog, const int32_t* pool, int c0,
                     int nq, const uint32_t** mask_out, int* qs_out, cudaStream_t st) {
  const int qs = std::max(32, next_pow2(nq));
  WhereChunk ch;
  where_plan_chunk(p_off, prog, pool, c0, nq, qs, ch);
  const size_t smem = where_chunk_smem(ch);
  SB_REQUIRE(smem <= ctx->smem_optin, SB_ERR_UNSUPPORTED, "dense: filter programs need %zu bytes of shared memory", smem);
  // device: counts [qs] | the chunk's programs | mask
  const size_t o_stage = align16((size_t)qs * 4);
  const size_t o_mask = (o_stage + ch.bytes.size() + 255) / 256 * 256;
  int rc;
  if ((rc = ctx->filt_dev.reserve(o_mask + (size_t)(ix.n_pad / 32) * qs * 4))) return rc;
  if ((rc = ctx->filt_pin.reserve(ch.bytes.size() + 16))) return rc;
  uint8_t* dv = ctx->filt_dev.as<uint8_t>();
  SB_CUDA(cudaStreamSynchronize(st));   // the pinned staging may still feed an earlier call's copies
  memcpy(ctx->filt_pin.p, ch.bytes.data(), ch.bytes.size());
  SB_CUDA(cudaMemcpyAsync(dv + o_stage, ctx->filt_pin.p, ch.bytes.size(), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemsetAsync(dv, 0, (size_t)qs * 4, st));
  SB_CUDA(cudaFuncSetAttribute(dense_where_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  uint32_t* mask = reinterpret_cast<uint32_t*>(dv + o_mask);
  if ((rc = where_mask_launches(ctx, ix, ch, dv + o_stage, mask, reinterpret_cast<int32_t*>(dv), qs, st))) return rc;
  *mask_out = mask;
  *qs_out = qs;
  return SB_OK;
}

namespace {

// Filtered top-k of B queries (q_pad on the device; one validated program per query, host arrays) in chunks of <= 256
// queries: per chunk the match mask + match counts, one wait for the counts, then the gather path for low-cardinality
// queries and the masked scans for the rest.  A batch of empty programs is the unfiltered search.
int dense_topk_where_enqueue(sb_ctx* ctx, DenseIndex& ix, const float* q_pad, int B, int k, const int32_t* p_off,
                             const sb_pred* prog, const int32_t* pool, int64_t* out_ids, double* out_scores,
                             int32_t* out_counts, cudaStream_t st) {
  SB_REQUIRE(k <= kDenseMaxK, SB_ERR_UNSUPPORTED, "dense: top_k %d too large (max %d per call)", k, kDenseMaxK);
  if (p_off[B] == 0)   // no query has a program: exactly the unfiltered search
    return dense_topk_enqueue(ctx, ix, q_pad, B, k, out_ids, out_scores, out_counts, st);

  const int64_t n_words = ix.n_pad / 32;
  int qchunk = 256;   // queries per mask; the mask (n_pad * qchunk / 8 bytes) is kept under 1 GB
  while (qchunk > 32 && (size_t)n_words * 4 * qchunk > (1ull << 30)) qchunk >>= 1;
  std::vector<WhereChunk> chunks((B + qchunk - 1) / qchunk);
  size_t stage_bytes = 0, smem_max = 0;
  for (size_t c = 0; c < chunks.size(); ++c) {
    const int c0 = (int)c * qchunk, nq = std::min(qchunk, B - c0);
    WhereChunk& ch = chunks[c];
    where_plan_chunk(p_off, prog, pool, c0, nq, std::max(32, next_pow2(nq)), ch);
    stage_bytes = std::max(stage_bytes, ch.bytes.size());
    smem_max = std::max(smem_max, where_chunk_smem(ch));
  }
  // device: counts [qchunk] | state [qchunk] | qlist [qchunk] | one chunk's programs | mask
  const size_t o_cnt = 0, o_state = (size_t)qchunk * 4, o_qlist = o_state + (size_t)qchunk * 4;
  const size_t o_stage = align16(o_qlist + (size_t)qchunk * 4);
  const size_t o_mask = (o_stage + stage_bytes + 255) / 256 * 256;
  const size_t dev_bytes = o_mask + (size_t)n_words * qchunk * 4;
  int rc;
  if ((rc = ctx->filt_dev.reserve(dev_bytes))) return rc;
  if ((rc = ctx->filt_pin.reserve(o_mask))) return rc;
  uint8_t* dv = ctx->filt_dev.as<uint8_t>();
  uint8_t* hp = ctx->filt_pin.as<uint8_t>();
  SB_CUDA(cudaStreamSynchronize(st));   // the pinned staging may still feed an earlier call's copies
  int32_t* cnt_h = reinterpret_cast<int32_t*>(hp + o_cnt);
  int32_t* state_h = reinterpret_cast<int32_t*>(hp + o_state);
  int32_t* qlist_h = reinterpret_cast<int32_t*>(hp + o_qlist);
  int32_t* cnt_d = reinterpret_cast<int32_t*>(dv + o_cnt);
  int32_t* state_d = reinterpret_cast<int32_t*>(dv + o_state);
  int32_t* qlist_d = reinterpret_cast<int32_t*>(dv + o_qlist);
  uint32_t* mask = reinterpret_cast<uint32_t*>(dv + o_mask);
  SB_REQUIRE(smem_max <= ctx->smem_optin, SB_ERR_UNSUPPORTED, "dense: filter programs need %zu bytes of shared memory",
             smem_max);
  SB_CUDA(cudaFuncSetAttribute(dense_where_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
  const size_t gather_smem = (size_t)kGatherMax * 20 + (size_t)ix.d_pad * 4 + 64;
  auto gather_kern = ix.storage == SB_STORAGE_U8    ? dense_filter_gather_kernel<SB_STORAGE_U8>
                     : ix.storage == SB_STORAGE_F32 ? dense_filter_gather_kernel<SB_STORAGE_F32>
                                                    : dense_filter_gather_kernel<SB_STORAGE_F16>;
  SB_CUDA(cudaFuncSetAttribute(gather_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gather_smem));
  for (int c0 = 0; c0 < B; c0 += qchunk) {
    const int nq = std::min(qchunk, B - c0);
    const int qs = std::max(32, next_pow2(nq));   // >= the widest wgmma group of the chunk
    const WhereChunk& ch = chunks[c0 / qchunk];
    memcpy(hp + o_stage, ch.bytes.data(), ch.bytes.size());
    SB_CUDA(cudaMemcpyAsync(dv + o_stage, hp + o_stage, ch.bytes.size(), cudaMemcpyHostToDevice, st));
    SB_CUDA(cudaMemsetAsync(cnt_d, 0, (size_t)qs * 4, st));
    if ((rc = where_mask_launches(ctx, ix, ch, dv + o_stage, mask, cnt_d, qs, st))) return rc;
    SB_CUDA(cudaMemcpyAsync(cnt_h, cnt_d, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    // route: a filtered query with <= kGatherMax matching rows is answered exactly from its matches; the others are
    // scanned with the mask (a query without a program matches every row)
    int n_gather = 0;
    int64_t c_min = ix.n;
    for (int q = 0; q < nq; ++q) {
      const bool filtered = p_off[c0 + q + 1] > p_off[c0 + q];
      const bool gather = filtered && cnt_h[q] <= kGatherMax;
      state_h[q] = gather ? 1 : 0;
      if (gather) qlist_h[n_gather++] = q;
      else c_min = std::min<int64_t>(c_min, cnt_h[q]);
    }
    SB_CUDA(cudaMemcpyAsync(state_d, state_h, (size_t)qchunk * 8, cudaMemcpyHostToDevice, st));  // state + qlist
    const float* qc = q_pad + (size_t)c0 * ix.d_pad;
    int64_t* oi = out_ids + (size_t)c0 * k;
    double* os = out_scores + (size_t)c0 * k;
    int32_t* oc = out_counts + c0;
    if (n_gather > 0) {
      GatherParams gp;
      gp.mask = mask;
      gp.qs = qs;
      gp.n_words = n_words;
      gp.qlist = qlist_d;
      gp.slot = slot_view(ix);
      gp.q = qc;
      gp.k = k;
      gp.out_ids = oi;
      gp.out_scores = os;
      gp.out_counts = oc;
      ProfScope ps(ctx, SB_PROF_DENSE_GATHER, st);
      gather_kern<<<n_gather, kMergeThreads, gather_smem, st>>>(gp);
    }
    SB_CUDA(cudaGetLastError());
    if (n_gather < nq) {
      DenseFilter flt;
      flt.mask = mask;
      flt.qs = qs;
      flt.state = state_d;
      flt.state_host = state_h;
      flt.c_min = c_min;
      if ((rc = dense_topk_enqueue(ctx, ix, qc, nq, k, oi, os, oc, st, &flt))) return rc;
    }
  }
  return SB_OK;
}


// Legacy conditions (CSR f_off / f_field / f_code, conjunctions of "tag == code") and grouped search's exclusion mode
// (x_field >= 0: the row's code at x_field must be present and absent from the query's ascending x_code range) as
// programs: per query the conjunction reduced to one EQ leaf per field (a negative code, or two codes on one field,
// match nothing: one empty IN leaf), then PRESENT(x) AND NOR(IN(x, codes)), under one AND.  Every query is filtered in
// exclusion mode; without it a query without conditions gets the empty program (unfiltered).
int dense_topk_filtered_enqueue(sb_ctx* ctx, DenseIndex& ix, const float* q_pad, int B, int k, const int32_t* f_off,
                                const int32_t* f_field, const int32_t* f_code, int64_t* out_ids, double* out_scores,
                                int32_t* out_counts, cudaStream_t st, int x_field = -1, const int32_t* x_off = nullptr,
                                const int32_t* x_code = nullptr) {
  SB_REQUIRE(f_off[0] == 0, SB_ERR_ARG, "sb_dense_topk_filtered: f_off[0] must be 0");
  for (int b = 0; b < B; ++b)
    SB_REQUIRE(f_off[b + 1] >= f_off[b], SB_ERR_ARG, "sb_dense_topk_filtered: f_off is not non-decreasing at %d", b);
  const int n_conds = f_off[B];
  for (int i = 0; i < n_conds; ++i) {
    const int f = f_field[i];
    SB_REQUIRE(f >= 0 && f < SB_MAX_TAG_FIELDS, SB_ERR_ARG, "sb_dense_topk_filtered: field %d out of range", f);
    SB_REQUIRE(ix.tags[f] != nullptr, SB_ERR_STATE, "sb_dense_topk_filtered: field %d has no tag column loaded", f);
  }
  std::vector<int32_t> p_off(B + 1, 0), pool;
  std::vector<sb_pred> prog;
  auto leaf = [&](int op, int field, int a, int b) {
    sb_pred e = {};
    e.op = op;
    e.field = field;
    e.a = a;
    e.b = b;
    prog.push_back(e);
  };
  for (int b = 0; b < B; ++b) {
    int32_t code_of[SB_MAX_TAG_FIELDS];
    std::fill(code_of, code_of + SB_MAX_TAG_FIELDS, -2);
    bool none = false;
    for (int i = f_off[b]; i < f_off[b + 1]; ++i) {
      const int f = f_field[i], c = f_code[i];
      none |= c < 0 || (code_of[f] != -2 && code_of[f] != c);
      code_of[f] = c;
    }
    if (none) {
      leaf(SB_PRED_IN, f_field[f_off[b]], 0, 0);
    } else {
      int n = 0;
      for (int f = 0; f < SB_MAX_TAG_FIELDS; ++f)
        if (code_of[f] >= 0) {
          leaf(SB_PRED_EQ, f, code_of[f], 0);
          ++n;
        }
      if (x_field >= 0) {
        leaf(SB_PRED_PRESENT, x_field, 0, 0);
        leaf(SB_PRED_IN, x_field, (int32_t)pool.size(), x_off[b + 1] - x_off[b]);
        pool.insert(pool.end(), x_code + x_off[b], x_code + x_off[b + 1]);
        leaf(SB_PRED_NOR, 0, 1, 0);
        n += 2;
      }
      if (n > 1) leaf(SB_PRED_AND, 0, n, 0);
    }
    p_off[b + 1] = (int32_t)prog.size();
  }
  return dense_topk_where_enqueue(ctx, ix, q_pad, B, k, p_off.data(), prog.data(), pool.data(), out_ids, out_scores,
                                  out_counts, st);
}

// Grouped search of B padded queries (DESIGN.md K1f) into ctx->grp_res_dev, laid out n_groups [B] | g_code [B][L] |
// g_hits [B][L] | h_ids [B][L][G] | h_scores [B][L][G] (offsets in *o).  Every step consumes an exact ordered prefix:
//   round 1      the exact top-K of the rows matching the query's conditions;
//   exclusion    while a query's prefix was full and it has fewer than L groups: the exact top-K of its matching rows
//                that have a group not found yet -- their first groups are the next groups in the ranking;
//   completion   a group found with fewer than G hits in a full prefix: the top-G of "conditions and group_by == code".
// f_off == nullptr: no conditions.  Inputs are validated by the caller.
struct GroupLayout {
  size_t n_groups, g_code, g_hits, h_ids, h_scores, total;
};

int dense_groups_enqueue(sb_ctx* ctx, DenseIndex& ix, const float* q_pad, int B, int gf, int L, int G,
                         const int32_t* f_off, const int32_t* f_field, const int32_t* f_code, GroupLayout* o,
                         cudaStream_t st) {
  const int K = std::min(kDenseMaxK, std::max(128, 4 * L * G));
  const size_t BL = (size_t)B * L, BLG = BL * G;
  o->n_groups = 0;
  o->g_code = align16((size_t)B * 4);
  o->g_hits = o->g_code + align16(BL * 4);
  o->h_ids = o->g_hits + align16(BL * 4);
  o->h_scores = o->h_ids + BLG * 8;
  o->total = o->h_scores + BLG * 8;
  int rc;
  if ((rc = ctx->grp_res_dev.reserve(o->total))) return rc;
  uint8_t* res = ctx->grp_res_dev.as<uint8_t>();
  int32_t* n_groups = reinterpret_cast<int32_t*>(res + o->n_groups);
  int32_t* g_code = reinterpret_cast<int32_t*>(res + o->g_code);
  int32_t* g_hits = reinterpret_cast<int32_t*>(res + o->g_hits);
  int64_t* h_ids = reinterpret_cast<int64_t*>(res + o->h_ids);
  double* h_scores = reinterpret_cast<double*>(res + o->h_scores);
  SB_CUDA(cudaMemsetAsync(n_groups, 0, (size_t)B * 4, st));
  SB_CUDA(cudaMemsetAsync(g_code, 0xff, BL * 4, st));
  SB_CUDA(cudaMemsetAsync(g_hits, 0, BL * 4, st));
  SB_CUDA(cudaMemsetAsync(h_ids, 0xff, BLG * 8, st));
  SB_CUDA(cudaMemsetAsync(h_scores, 0, BLG * 8, st));
  // one round: prefixes ids [B][K] | scores [B][K] | counts [B] | qmap [B]
  const size_t r_sc = (size_t)B * K * 8, r_cnt = r_sc + (size_t)B * K * 8, r_map = r_cnt + align16((size_t)B * 4);
  if ((rc = ctx->grp_round_dev.reserve(r_map + (size_t)B * 4))) return rc;
  uint8_t* rd = ctx->grp_round_dev.as<uint8_t>();
  int64_t* rids = reinterpret_cast<int64_t*>(rd);
  double* rsc = reinterpret_cast<double*>(rd + r_sc);
  int32_t* rcnt = reinterpret_cast<int32_t*>(rd + r_cnt);
  int32_t* rmap = reinterpret_cast<int32_t*>(rd + r_map);
  const int32_t* tag = ix.tags[gf];

  GroupCollectParams cp;
  cp.ids = rids;
  cp.scores = rsc;
  cp.counts = rcnt;
  cp.tag = tag;
  cp.id_base = ix.id_base;
  cp.K = K;
  cp.L = L;
  cp.G = G;
  cp.n_groups = n_groups;
  cp.g_code = g_code;
  cp.g_hits = g_hits;
  cp.h_ids = h_ids;
  cp.h_scores = h_scores;

  std::vector<int32_t> qmap(B), cnt_h(B), ng_h(B), prev(B, 0), rounds(B, 1), code_h(BL), hits_h(BL);
  for (int b = 0; b < B; ++b) qmap[b] = b;
  std::vector<int32_t> incomplete;   // b * L + g
  auto no_conds = [&](int b) { return f_off == nullptr || f_off[b + 1] == f_off[b]; };
  int nq = B;
  for (int round = 0; nq > 0; ++round) {
    if (round == 0) {
      if (f_off == nullptr) rc = dense_topk_enqueue(ctx, ix, q_pad, B, K, rids, rsc, rcnt, st);
      else rc = dense_topk_filtered_enqueue(ctx, ix, q_pad, B, K, f_off, f_field, f_code, rids, rsc, rcnt, st);
      if (rc) return rc;
      cp.qmap = nullptr;
    } else {
      // the short queries' conditions, and their groups found so far (ascending) as the exclusion list
      std::vector<int32_t> off(nq + 1, 0), fld, code, xoff(nq + 1, 0), xcode;
      for (int i = 0; i < nq; ++i) {
        const int b = qmap[i];
        if (!no_conds(b))
          for (int j = f_off[b]; j < f_off[b + 1]; ++j) {
            fld.push_back(f_field[j]);
            code.push_back(f_code[j]);
          }
        off[i + 1] = (int32_t)fld.size();
        const size_t x0 = xcode.size();
        xcode.insert(xcode.end(), code_h.begin() + (size_t)b * L, code_h.begin() + (size_t)b * L + ng_h[b]);
        std::sort(xcode.begin() + x0, xcode.end());
        xoff[i + 1] = (int32_t)xcode.size();
      }
      if ((rc = ctx->grp_q_dev.reserve((size_t)nq * ix.d_pad * 4))) return rc;
      float* qr = ctx->grp_q_dev.as<float>();
      SB_CUDA(cudaMemcpyAsync(rmap, qmap.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st));
      ctx->launches += 1;
      dense_group_queries_kernel<<<nq, 256, 0, st>>>(q_pad, rmap, ix.d_pad, qr);
      SB_CUDA(cudaGetLastError());
      if ((rc = dense_topk_filtered_enqueue(ctx, ix, qr, nq, K, off.data(), fld.data(), code.data(), rids, rsc, rcnt, st,
                                            gf, xoff.data(), xcode.data())))
        return rc;
      cp.qmap = rmap;
    }
    {
      ProfScope ps(ctx, SB_PROF_DENSE_GROUP_COLLECT, st);
      dense_group_collect_kernel<<<nq, kGroupThreads, 0, st>>>(cp);
    }
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaMemcpyAsync(cnt_h.data(), rcnt, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(ng_h.data(), n_groups, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(code_h.data(), g_code, BL * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(hits_h.data(), g_hits, BL * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    // a full prefix proves nothing past its end: its groups short of G hits need completion, and a query short of L
    // groups goes on to an exclusion round.  A prefix that is not full held every remaining matching row.
    int next = 0;
    for (int i = 0; i < nq; ++i) {
      const int b = qmap[i];
      if (cnt_h[i] < K) continue;
      for (int g = prev[b]; g < ng_h[b]; ++g)
        if (hits_h[(size_t)b * L + g] < G) incomplete.push_back((int32_t)((size_t)b * L + g));
      prev[b] = ng_h[b];
      if (ng_h[b] < L) {
        qmap[next++] = b;
        rounds[b] += 1;
      }
    }
    nq = next;
  }
  for (int b = 0; b < B; ++b) {
    const size_t r = (size_t)rounds[b] - 1;
    if (ctx->grp_rounds.size() <= r) ctx->grp_rounds.resize(r + 1, 0);
    ctx->grp_rounds[r] += 1;
  }

  const int np = (int)incomplete.size();
  if (np == 0) return SB_OK;
  std::vector<int32_t> src(np), off(np + 1, 0), fld, code;
  for (int i = 0; i < np; ++i) {
    const int b = incomplete[i] / L;
    src[i] = b;
    if (!no_conds(b))
      for (int j = f_off[b]; j < f_off[b + 1]; ++j) {
        fld.push_back(f_field[j]);
        code.push_back(f_code[j]);
      }
    fld.push_back(gf);
    code.push_back(code_h[incomplete[i]]);
    off[i + 1] = (int32_t)fld.size();
  }
  // completions: ids [np][G] | scores [np][G] | counts [np] | src [np] | dest [np]
  const size_t c_sc = (size_t)np * G * 8, c_cnt = c_sc + (size_t)np * G * 8, c_src = c_cnt + align16((size_t)np * 4);
  const size_t c_dst = c_src + align16((size_t)np * 4);
  if ((rc = ctx->grp_cmp_dev.reserve(c_dst + (size_t)np * 4))) return rc;
  if ((rc = ctx->grp_q_dev.reserve((size_t)np * ix.d_pad * 4))) return rc;
  uint8_t* cd = ctx->grp_cmp_dev.as<uint8_t>();
  int32_t* src_d = reinterpret_cast<int32_t*>(cd + c_src);
  int32_t* dst_d = reinterpret_cast<int32_t*>(cd + c_dst);
  float* qr = ctx->grp_q_dev.as<float>();
  SB_CUDA(cudaMemcpyAsync(src_d, src.data(), (size_t)np * 4, cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemcpyAsync(dst_d, incomplete.data(), (size_t)np * 4, cudaMemcpyHostToDevice, st));
  ctx->launches += 1;
  dense_group_queries_kernel<<<np, 256, 0, st>>>(q_pad, src_d, ix.d_pad, qr);
  SB_CUDA(cudaGetLastError());
  GroupAssembleParams ap;
  ap.ids = reinterpret_cast<int64_t*>(cd);
  ap.scores = reinterpret_cast<double*>(cd + c_sc);
  ap.counts = reinterpret_cast<int32_t*>(cd + c_cnt);
  if ((rc = dense_topk_filtered_enqueue(ctx, ix, qr, np, G, off.data(), fld.data(), code.data(),
                                        const_cast<int64_t*>(ap.ids), const_cast<double*>(ap.scores),
                                        const_cast<int32_t*>(ap.counts), st)))
    return rc;
  ap.dest = dst_d;
  ap.G = G;
  ap.n = (int64_t)np * G;
  ap.g_hits = g_hits;
  ap.h_ids = h_ids;
  ap.h_scores = h_scores;
  {
    ProfScope ps(ctx, SB_PROF_DENSE_GROUP_ASSEMBLE, st);
    dense_group_assemble_kernel<<<(unsigned)((ap.n + 255) / 256), 256, 0, st>>>(ap);
  }
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int64_t round_rows(int64_t n) { return (n + kRowPad - 1) / kRowPad * kRowPad; }

// The one store-rows path of sb_dense_load and sb_dense_upsert: n host rows (SB_F32 / SB_F16) through a device staging
// buffer in chunks, converted by dense_store_rows_kernel into rows row0 + i, or dst_dev[i] (a device list) when given.
// A float32 slot also gets rows32 from dense_store_rows32_kernel, and *sigma the largest sigma of the stored rows.  A
// uint8 slot is written by dense_store_rows8_kernel alone (SB_U8 / SB_F32 / SB_F16 input, checked by check_u8_rows), and
// *sigma receives the largest ||x||^2 of the stored rows instead.  Returns after the last chunk has been stored.
int dense_store_staged(sb_ctx* ctx, DenseIndex& ix, const void* vecs, int64_t n, int32_t dtype, const int64_t* dst_dev,
                       int64_t row0, double* sigma) {
  const int d = ix.d;
  const size_t esz = dtype == SB_F32 ? 4 : dtype == SB_U8 ? 1 : 2;
  const bool u8 = ix.storage == SB_STORAGE_U8, f32 = ix.storage == SB_STORAGE_F32;
  const int64_t chunk_rows = std::max<int64_t>(1, (int64_t)((256ull << 20) / ((size_t)d * esz)));
  int rc = ctx->misc_dev.reserve((size_t)std::min<int64_t>(chunk_rows, n) * d * esz);
  if (rc) return rc;
  unsigned long long* sigma_bits = nullptr;
  if (f32 || u8) {
    if ((rc = ctx->sigma_dev.reserve(8))) return rc;
    sigma_bits = ctx->sigma_dev.as<unsigned long long>();
    SB_CUDA(cudaMemsetAsync(sigma_bits, 0, 8, ctx->stream));
  }
  for (int64_t r0 = 0; r0 < n; r0 += chunk_rows) {
    const int64_t nr = std::min<int64_t>(chunk_rows, n - r0);
    const uint8_t* src = reinterpret_cast<const uint8_t*>(vecs) + (size_t)r0 * d * esz;
    SB_CUDA(cudaMemcpyAsync(ctx->misc_dev.p, src, (size_t)nr * d * esz, cudaMemcpyHostToDevice, ctx->stream));
    const int wpb = 8;
    const unsigned blocks = (unsigned)((nr + wpb - 1) / wpb);
    const int64_t* dst = dst_dev ? dst_dev + r0 : nullptr;
    if (u8) {
      const bool cos = ix.metric == SB_METRIC_COSINE;
      if (dtype == SB_U8)
        dense_store_rows8_kernel<uint8_t><<<blocks, wpb * 32, 0, ctx->stream>>>(
            ctx->misc_dev.as<uint8_t>(), nr, d, ix.d_pad, ix.rows8, ix.inv_norm, row0 + r0, dst, cos, ix.hh, sigma_bits);
      else if (dtype == SB_F32)
        dense_store_rows8_kernel<float><<<blocks, wpb * 32, 0, ctx->stream>>>(
            ctx->misc_dev.as<float>(), nr, d, ix.d_pad, ix.rows8, ix.inv_norm, row0 + r0, dst, cos, ix.hh, sigma_bits);
      else
        dense_store_rows8_kernel<__half><<<blocks, wpb * 32, 0, ctx->stream>>>(
            ctx->misc_dev.as<__half>(), nr, d, ix.d_pad, ix.rows8, ix.inv_norm, row0 + r0, dst, cos, ix.hh, sigma_bits);
    } else if (dtype == SB_F32)
      dense_store_rows_kernel<float><<<blocks, wpb * 32, 0, ctx->stream>>>(ctx->misc_dev.as<float>(), nr, d, ix.d_pad,
                                                                           ix.rows, ix.inv_norm, row0 + r0, dst, true,
                                                                           ix.cfac, ix.hh);
    else   // Cosine keeps fp16 input verbatim; Dot / Euclid normalise it like fp32 input
      dense_store_rows_kernel<__half><<<blocks, wpb * 32, 0, ctx->stream>>>(ctx->misc_dev.as<__half>(), nr, d, ix.d_pad,
                                                                            ix.rows, ix.inv_norm, row0 + r0, dst,
                                                                            ix.cfac != nullptr, ix.cfac, ix.hh);
    SB_CUDA(cudaGetLastError());
    if (f32) {
      if (dtype == SB_F32)
        dense_store_rows32_kernel<float><<<blocks, wpb * 32, 0, ctx->stream>>>(
            ctx->misc_dev.as<float>(), nr, d, ix.d_pad, ix.rows, ix.rows32, row0 + r0, dst, ix.cfac, sigma_bits);
      else
        dense_store_rows32_kernel<__half><<<blocks, wpb * 32, 0, ctx->stream>>>(
            ctx->misc_dev.as<__half>(), nr, d, ix.d_pad, ix.rows, ix.rows32, row0 + r0, dst, ix.cfac, sigma_bits);
      SB_CUDA(cudaGetLastError());
    }
    SB_CUDA(cudaStreamSynchronize(ctx->stream));  // staging buffer is reused by the next chunk
  }
  *sigma = 0.0;
  if (sigma_bits) {
    unsigned long long bits = 0;
    SB_CUDA(cudaMemcpy(&bits, sigma_bits, 8, cudaMemcpyDeviceToHost));
    if (u8) *sigma = (double)bits;   // an integer ||x||^2, not fp64 bits
    else memcpy(sigma, &bits, 8);
  }
  return SB_OK;
}

// One per-row device column of a slot: the address of its pointer field in DenseIndex, its bytes per row and the byte
// its unused capacity [n, n_cap) holds.
struct DenseColumn {
  void** ptr;
  int32_t row_bytes;
  int fill;
};

template <typename T>
DenseColumn column(T*& field, int32_t row_bytes, int fill) {
  return {reinterpret_cast<void**>(&field), row_bytes, fill};
}
DenseColumn tag_column(DenseIndex& ix, int f) { return column(ix.tags[f], 4, 0xff); }     // code -1
DenseColumn value_column(DenseIndex& ix, int f) { return column(ix.vals[f], 8, 0xff); }   // NaN

// The columns a slot has, from its storage, metric and loaded payload fields.  Every one spans n_cap rows (a payload
// column loaded on an empty slot: 1 row).  Returns their count (<= kMaxDenseColumns).
int dense_columns(DenseIndex& ix, DenseColumn* out) {
  int n = 0;
  if (ix.storage == SB_STORAGE_U8) out[n++] = column(ix.rows8, ix.d_pad, 0);
  else out[n++] = column(ix.rows, 2 * ix.d_pad, 0);
  if (ix.storage == SB_STORAGE_F32) out[n++] = column(ix.rows32, 4 * ix.d_pad, 0);
  out[n++] = column(ix.inv_norm, 4, 0);
  if (ix.metric != SB_METRIC_COSINE && ix.storage != SB_STORAGE_U8) out[n++] = column(ix.cfac, 8, 0);
  if (ix.metric == SB_METRIC_EUCLID) out[n++] = column(ix.hh, 4, 0);
  for (int f = 0; f < SB_MAX_TAG_FIELDS; ++f)
    if (ix.tags[f]) out[n++] = tag_column(ix, f);
  for (int f = 0; f < SB_MAX_VALUE_FIELDS; ++f)
    if (ix.vals[f]) out[n++] = value_column(ix, f);
  return n;
}

// *p = `rows` rows of column c, rows [from, rows) filled (stream-ordered on st)
cudaError_t column_alloc(const DenseColumn& c, void** p, int64_t rows, int64_t from, cudaStream_t st) {
  cudaError_t e = cudaMalloc(p, (size_t)rows * c.row_bytes);
  if (e != cudaSuccess) return e;
  return cudaMemsetAsync(static_cast<uint8_t*>(*p) + (size_t)from * c.row_bytes, c.fill,
                         (size_t)(rows - from) * c.row_bytes, st);
}

// Reallocate every column to n_cap rows (> ix.n_cap): the [0, n_pad) prefix is copied device to device, the rest is
// filled.  The old buffers stay valid until every new one is complete; on failure the slot is unchanged.
int dense_grow(sb_ctx* ctx, DenseIndex& ix, int64_t n_cap) {
  DenseColumn col[kMaxDenseColumns];
  const int nc = dense_columns(ix, col);
  void* fresh[kMaxDenseColumns] = {};
  const int64_t keep = ix.n_pad;
  cudaStream_t st = ctx->stream;
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < nc && e == cudaSuccess; ++i) {
    e = column_alloc(col[i], &fresh[i], n_cap, keep, st);
    if (e == cudaSuccess && keep)
      e = cudaMemcpyAsync(fresh[i], *col[i].ptr, (size_t)keep * col[i].row_bytes, cudaMemcpyDeviceToDevice, st);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {   // the slot keeps its old buffers; the new ones are released on every failure
    cudaStreamSynchronize(st);
    for (int i = 0; i < nc; ++i) cudaFree(fresh[i]);
    sb_set_error("dense: growing slot to %lld rows failed: %s", (long long)n_cap, cudaGetErrorString(e));
    return SB_ERR_CUDA;
  }
  for (int i = 0; i < nc; ++i) {
    cudaFree(*col[i].ptr);
    *col[i].ptr = fresh[i];
  }
  ix.n_cap = n_cap;
  return SB_OK;
}

// (Re)load payload column c with rows[0, n) (n = the slot's row count).  It spans the slot's capacity, at least one
// row, so upserts and deletes never reallocate it alone.
int dense_payload_load(sb_ctx* ctx, DenseIndex& ix, const DenseColumn& c, const void* rows, int64_t n) {
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  cudaFree(*c.ptr);
  *c.ptr = nullptr;
  SB_CUDA(column_alloc(c, c.ptr, std::max<int64_t>(ix.n_cap, 1), n, ctx->stream));
  if (n) SB_CUDA(cudaMemcpyAsync(*c.ptr, rows, (size_t)n * c.row_bytes, cudaMemcpyHostToDevice, ctx->stream));
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  return SB_OK;
}

// rows[0..n) all in [0, limit) and pairwise distinct; `sorted` receives them in ascending order
int check_rows(const char* who, const int64_t* rows, int64_t n, int64_t limit, std::vector<int64_t>& sorted) {
  sorted.assign(rows, rows + n);
  std::sort(sorted.begin(), sorted.end());
  for (int64_t i = 0; i < n; ++i) {
    SB_REQUIRE(sorted[i] >= 0 && sorted[i] < limit, SB_ERR_ARG, "%s: row %lld out of range [0, %lld)", who,
               (long long)sorted[i], (long long)limit);
    SB_REQUIRE(i == 0 || sorted[i] != sorted[i - 1], SB_ERR_ARG, "%s: row %lld given twice", who, (long long)sorted[i]);
  }
  return SB_OK;
}

// Dot / Euclid input rows, checked on the host before anything changes: every fp64 norm finite and, for Euclid, every
// squared norm finite in fp32.  Returns the norm bounds the rows need: *rho >= max ||v||, *hmax >= max h (DESIGN.md K1e;
// the device sums in another order, which the 2^-20 margin covers many times over).
int check_metric_rows(const char* who, int metric, const void* vecs, int64_t n, int d, int32_t dtype, double* rho,
                      double* hmax) {
  double mx = 0.0;
  for (int64_t r = 0; r < n; ++r) {
    double ss = 0.0;
    if (dtype == SB_F32) {
      const float* v = reinterpret_cast<const float*>(vecs) + (size_t)r * d;
      for (int i = 0; i < d; ++i) ss += (double)v[i] * (double)v[i];
    } else {
      const __half* v = reinterpret_cast<const __half*>(vecs) + (size_t)r * d;
      for (int i = 0; i < d; ++i) {
        const double x = (double)__half2float(v[i]);
        ss += x * x;
      }
    }
    SB_REQUIRE(std::isfinite(ss), SB_ERR_ARG, "%s: row %lld has a non-finite norm", who, (long long)r);
    SB_REQUIRE(metric != SB_METRIC_EUCLID || ss <= (double)FLT_MAX, SB_ERR_ARG,
               "%s: row %lld has a squared norm %g beyond the fp32 range (Euclid)", who, (long long)r, ss);
    mx = std::max(mx, ss);
  }
  const double m = 1.0 + 0x1p-20;
  *rho = sqrt(mx) * m;
  const double hv = 0.5 * mx * m;
  float hf = (float)hv;
  if ((double)hf < hv) hf = nextafterf(hf, INFINITY);
  *hmax = metric == SB_METRIC_EUCLID ? (double)hf : 0.0;
  return SB_OK;
}

// Input rows of a uint8 slot, checked on the host before anything changes: every value an integer in [0, 255].  SB_U8
// input holds nothing else.
int check_u8_rows(const char* who, const void* vecs, int64_t n, int d, int32_t dtype) {
  if (dtype == SB_U8) return SB_OK;
  for (int64_t r = 0; r < n; ++r)
    for (int i = 0; i < d; ++i) {
      const size_t at = (size_t)r * d + i;
      const float v = dtype == SB_F32 ? reinterpret_cast<const float*>(vecs)[at]
                                      : __half2float(reinterpret_cast<const __half*>(vecs)[at]);
      SB_REQUIRE(v >= 0.f && v <= 255.f && v == floorf(v), SB_ERR_ARG,
                 "%s: row %lld, component %d is %g; a uint8 slot takes integers in [0, 255]", who, (long long)r, i,
                 (double)v);
    }
  return SB_OK;
}

// rho >= max ||x|| and hmax >= max ||x||^2 / 2 (rounded up to fp32, as hh is) of uint8 rows whose largest ||x||^2 is xx
void u8_norm_bounds(int metric, double xx, double* rho, double* hmax) {
  *rho = metric == SB_METRIC_COSINE ? 0.0 : sqrt(xx) * (1.0 + 0x1p-20);
  float hf = (float)(0.5 * xx);
  if ((double)hf < 0.5 * xx) hf = nextafterf(hf, INFINITY);
  *hmax = metric == SB_METRIC_EUCLID ? (double)hf : 0.0;
}

}  // namespace

// Frees every column of the slot (sb_dense_load, sb_destroy).
void dense_free(DenseIndex& ix) {
  DenseColumn col[kMaxDenseColumns];
  const int nc = dense_columns(ix, col);
  for (int i = 0; i < nc; ++i) cudaFree(*col[i].ptr);
}

// Shared with other translation units (hybrid batch path, scorers).
int sb_dense_pad_queries(sb_ctx* ctx, const DenseIndex& ix, const float* q, int B, bool q_on_device, float** q_pad_out,
                         cudaStream_t st) {
  int rc = ctx->q_dev.reserve((size_t)B * ix.d_pad * sizeof(float));
  if (rc) return rc;
  float* qp = ctx->q_dev.as<float>();
  if (ix.d_pad != ix.d) SB_CUDA(cudaMemsetAsync(qp, 0, (size_t)B * ix.d_pad * sizeof(float), st));
  SB_CUDA(cudaMemcpy2DAsync(qp, (size_t)ix.d_pad * sizeof(float), q, (size_t)ix.d * sizeof(float),
                            (size_t)ix.d * sizeof(float), (size_t)B,
                            q_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
  *q_pad_out = qp;
  return SB_OK;
}

extern "C" {

int sb_dense_load_storage(sb_ctx* ctx, int slot, const void* vecs, int64_t n, int32_t d, int32_t dtype, int64_t id_base,
                          int32_t metric, int32_t storage) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_load: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_load: bad slot %d", slot);
  SB_REQUIRE(n >= 0 && d > 0 && d <= 4096, SB_ERR_ARG, "sb_dense_load: bad shape n=%lld d=%d", (long long)n, d);
  SB_REQUIRE(n < (1ll << 31), SB_ERR_ARG, "sb_dense_load: a shard holds at most 2^31-1 rows");
  SB_REQUIRE(dtype == SB_F32 || dtype == SB_F16 || (dtype == SB_U8 && storage == SB_STORAGE_U8), SB_ERR_ARG,
             "sb_dense_load: dtype must be SB_F32 or SB_F16 (or SB_U8 for SB_STORAGE_U8)");
  SB_REQUIRE(n == 0 || vecs != nullptr, SB_ERR_ARG, "sb_dense_load: vecs is NULL");
  SB_REQUIRE(metric == SB_METRIC_COSINE || metric == SB_METRIC_DOT || metric == SB_METRIC_EUCLID, SB_ERR_ARG,
             "sb_dense_load: metric %d is not supported (SB_METRIC_COSINE, SB_METRIC_DOT or SB_METRIC_EUCLID)", metric);
  SB_REQUIRE(storage == SB_STORAGE_F16 || storage == SB_STORAGE_F32 || storage == SB_STORAGE_U8, SB_ERR_ARG,
             "sb_dense_load: storage %d is not supported (SB_STORAGE_F16, SB_STORAGE_F32 or SB_STORAGE_U8)", storage);
  const bool u8 = storage == SB_STORAGE_U8;
  double rho = 0.0, hmax = 0.0;
  if (u8) {   // the norm bounds come from the store kernel
    int rc = check_u8_rows("sb_dense_load", vecs, n, d, dtype);
    if (rc) return rc;
  } else if (metric != SB_METRIC_COSINE || storage == SB_STORAGE_F32) {   // float32 storage: finite norms for every metric
    int rc = check_metric_rows("sb_dense_load", metric, vecs, n, d, dtype, &rho, &hmax);
    if (rc) return rc;
    if (metric == SB_METRIC_COSINE) rho = 0.0;
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  DenseIndex& ix = ctx->dense[slot];
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  dense_free(ix);   // payload columns included: a load drops them
  ix = DenseIndex();
  ix.n = n;
  ix.d = d;
  ix.d_pad = u8 ? (d + 63) / 64 * 64 : (d + 7) / 8 * 8;   // uint8: 64-byte rows, every slot fits the wgmma scan
  ix.n_pad = round_rows(n);
  ix.id_base = id_base;
  ix.metric = metric;
  ix.storage = storage;
  ix.rho_max = rho;
  ix.h_max = hmax;
  if (n == 0) return SB_OK;   // an empty slot allocates nothing: its first growth allocates every column
  ix.n_cap = ix.n_pad;
  DenseColumn col[kMaxDenseColumns];
  const int nc = dense_columns(ix, col);
  for (int i = 0; i < nc; ++i) SB_CUDA(column_alloc(col[i], col[i].ptr, ix.n_cap, 0, ctx->stream));
  if (u8) {
    double xx = 0.0;
    int rc = dense_store_staged(ctx, ix, vecs, n, dtype, nullptr, 0, &xx);
    u8_norm_bounds(metric, xx, &ix.rho_max, &ix.h_max);
    return rc;
  }
  return dense_store_staged(ctx, ix, vecs, n, dtype, nullptr, 0, &ix.sigma_max);
}

int sb_dense_load_metric(sb_ctx* ctx, int slot, const void* vecs, int64_t n, int32_t d, int32_t dtype, int64_t id_base,
                         int32_t metric) {
  return sb_dense_load_storage(ctx, slot, vecs, n, d, dtype, id_base, metric, SB_STORAGE_F16);
}

int sb_dense_load(sb_ctx* ctx, int slot, const void* vecs, int64_t n, int32_t d, int32_t dtype, int64_t id_base) {
  return sb_dense_load_metric(ctx, slot, vecs, n, d, dtype, id_base, SB_METRIC_COSINE);
}

int32_t sb_dense_metric(sb_ctx* ctx, int slot) {
  if (!ctx || slot < 0 || slot >= SB_MAX_DENSE_SLOTS) return -1;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return ctx->dense[slot].metric;
}

int32_t sb_dense_storage(sb_ctx* ctx, int slot) {
  if (!ctx || slot < 0 || slot >= SB_MAX_DENSE_SLOTS) return -1;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return ctx->dense[slot].storage;
}

int sb_dense_reserve(sb_ctx* ctx, int slot, int64_t n_cap) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_reserve: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_reserve: bad slot %d", slot);
  SB_REQUIRE(n_cap >= 0 && n_cap < (1ll << 31), SB_ERR_ARG, "sb_dense_reserve: bad capacity %lld", (long long)n_cap);
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_reserve: dense slot %d has no index loaded", slot);
  const int64_t want = round_rows(n_cap);
  if (want <= ix.n_cap) return SB_OK;
  SB_CUDA(cudaDeviceSynchronize());   // searches enqueued on other streams may still read the old buffers
  return dense_grow(ctx, ix, want);
}

int sb_dense_upsert(sb_ctx* ctx, int slot, const int64_t* rows, const void* vecs, int64_t n, int32_t dtype) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_upsert: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_upsert: bad slot %d", slot);
  SB_REQUIRE(n >= 0, SB_ERR_ARG, "sb_dense_upsert: bad n=%lld", (long long)n);
  SB_REQUIRE(dtype == SB_F32 || dtype == SB_F16 || dtype == SB_U8, SB_ERR_ARG,
             "sb_dense_upsert: dtype must be SB_F32, SB_F16 or SB_U8");
  SB_REQUIRE(n == 0 || (rows != nullptr && vecs != nullptr), SB_ERR_ARG, "sb_dense_upsert: NULL buffer");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_upsert: dense slot %d has no index loaded", slot);
  if (n == 0) return SB_OK;
  // rows < count overwrite; the others must be exactly count .. count + m - 1
  SB_REQUIRE(n < (1ll << 31) && ix.n + n < (1ll << 31), SB_ERR_ARG, "sb_dense_upsert: a shard holds at most 2^31-1 rows");
  std::vector<int64_t> sorted;
  int rc = check_rows("sb_dense_upsert", rows, n, ix.n + n, sorted);
  if (rc) return rc;
  const int64_t m = sorted.end() - std::lower_bound(sorted.begin(), sorted.end(), ix.n);
  SB_REQUIRE(m == 0 || (sorted[n - m] == ix.n && sorted[n - 1] == ix.n + m - 1), SB_ERR_ARG,
             "sb_dense_upsert: appended rows must be exactly %lld .. %lld", (long long)ix.n, (long long)(ix.n + m - 1));
  const bool u8 = ix.storage == SB_STORAGE_U8;
  SB_REQUIRE(dtype != SB_U8 || u8, SB_ERR_ARG, "sb_dense_upsert: SB_U8 rows need a uint8 slot");
  double rho = 0.0, hmax = 0.0, sigma = 0.0;
  if (u8) {
    if ((rc = check_u8_rows("sb_dense_upsert", vecs, n, ix.d, dtype))) return rc;
  } else if (ix.metric != SB_METRIC_COSINE || ix.storage == SB_STORAGE_F32) {
    if ((rc = check_metric_rows("sb_dense_upsert", ix.metric, vecs, n, ix.d, dtype, &rho, &hmax))) return rc;
    if (ix.metric == SB_METRIC_COSINE) rho = 0.0;
  }
  SB_CUDA(cudaDeviceSynchronize());   // searches enqueued on other streams may still read the slot
  const int64_t n_new = ix.n + m;
  if (round_rows(n_new) > ix.n_cap)
    if ((rc = dense_grow(ctx, ix, std::max(round_rows(n_new), round_rows(ix.n_cap + ix.n_cap / 2))))) return rc;
  if ((rc = ctx->misc2_dev.reserve((size_t)n * 8))) return rc;
  int64_t* dst = ctx->misc2_dev.as<int64_t>();
  SB_CUDA(cudaMemcpyAsync(dst, rows, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = dense_store_staged(ctx, ix, vecs, n, dtype, dst, 0, &sigma))) return rc;
  if (u8) {   // sigma is the largest ||x||^2 of the rows; a uint8 slot's own sigma stays 0
    u8_norm_bounds(ix.metric, sigma, &rho, &hmax);
    sigma = 0.0;
  }
  for (int f = 0; f < SB_MAX_TAG_FIELDS; ++f)
    if (ix.tags[f])
      dense_tags_scatter_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(ix.tags[f], dst, nullptr, n);
  for (int f = 0; f < SB_MAX_VALUE_FIELDS; ++f)
    if (ix.vals[f])
      dense_values_scatter_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(ix.vals[f], dst, nullptr, n);
  SB_CUDA(cudaGetLastError());
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  ix.n = n_new;
  ix.n_pad = round_rows(n_new);
  // the bounds only rise: an overwritten or deleted row's larger norm leaves a stale bound, which is still a bound
  ix.rho_max = std::max(ix.rho_max, rho);
  ix.h_max = std::max(ix.h_max, hmax);
  ix.sigma_max = std::max(ix.sigma_max, sigma);
  return SB_OK;
}

int sb_dense_tags_write(sb_ctx* ctx, int slot, int32_t field, const int64_t* rows, const int32_t* codes, int64_t n) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_tags_write: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_tags_write: bad slot %d", slot);
  SB_REQUIRE(field >= 0 && field < SB_MAX_TAG_FIELDS, SB_ERR_ARG, "sb_dense_tags_write: field %d out of range [0,%d)",
             field, SB_MAX_TAG_FIELDS);
  SB_REQUIRE(n >= 0, SB_ERR_ARG, "sb_dense_tags_write: bad n=%lld", (long long)n);
  SB_REQUIRE(n == 0 || (rows != nullptr && codes != nullptr), SB_ERR_ARG, "sb_dense_tags_write: NULL buffer");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_tags_write: dense slot %d has no index loaded", slot);
  SB_REQUIRE(ix.tags[field] != nullptr, SB_ERR_STATE, "sb_dense_tags_write: field %d has no tag column loaded", field);
  std::vector<int64_t> sorted;
  int rc = check_rows("sb_dense_tags_write", rows, n, ix.n, sorted);
  if (rc) return rc;
  for (int64_t i = 0; i < n; ++i)
    SB_REQUIRE(codes[i] >= -1, SB_ERR_ARG, "sb_dense_tags_write: code %d at entry %lld (must be >= -1)", codes[i],
               (long long)i);
  if (n == 0) return SB_OK;
  SB_CUDA(cudaDeviceSynchronize());
  if ((rc = ctx->misc2_dev.reserve((size_t)n * 12))) return rc;
  int64_t* r_dev = ctx->misc2_dev.as<int64_t>();
  int32_t* c_dev = reinterpret_cast<int32_t*>(r_dev + n);
  SB_CUDA(cudaMemcpyAsync(r_dev, rows, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  SB_CUDA(cudaMemcpyAsync(c_dev, codes, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  dense_tags_scatter_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(ix.tags[field], r_dev, c_dev, n);
  SB_CUDA(cudaGetLastError());
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  return SB_OK;
}

int sb_dense_delete(sb_ctx* ctx, int slot, const int64_t* rows, int64_t n, int64_t* moved_from, int64_t* moved_to,
                    int64_t* n_moved) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_delete: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_delete: bad slot %d", slot);
  SB_REQUIRE(n >= 0 && n_moved != nullptr, SB_ERR_ARG, "sb_dense_delete: bad arguments");
  SB_REQUIRE(n == 0 || (rows != nullptr && moved_from != nullptr && moved_to != nullptr), SB_ERR_ARG,
             "sb_dense_delete: NULL buffer");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_delete: dense slot %d has no index loaded", slot);
  std::vector<int64_t> del;
  int rc = check_rows("sb_dense_delete", rows, n, ix.n, del);
  if (rc) return rc;
  *n_moved = 0;
  if (n == 0) return SB_OK;
  // the plan: the surviving rows of the tail [keep, n), ascending, fill the deleted rows below `keep`, ascending
  const int64_t keep = ix.n - n;
  const int64_t n_holes = std::lower_bound(del.begin(), del.end(), keep) - del.begin();
  int64_t j = n_holes, src = keep, mv = 0;
  for (int64_t i = 0; i < n_holes; ++i, ++src) {
    while (j < n && del[j] == src) { ++j; ++src; }
    moved_from[mv] = src;
    moved_to[mv] = del[i];
    ++mv;
  }
  *n_moved = mv;
  SB_CUDA(cudaDeviceSynchronize());   // searches enqueued on other streams may still read the rows that move
  DenseColumn col[kMaxDenseColumns];
  const int nc = dense_columns(ix, col);
  if (mv) {
    if ((rc = ctx->misc2_dev.reserve((size_t)mv * 16))) return rc;
    int64_t* f_dev = ctx->misc2_dev.as<int64_t>();
    SB_CUDA(cudaMemcpyAsync(f_dev, moved_from, (size_t)mv * 8, cudaMemcpyHostToDevice, ctx->stream));
    SB_CUDA(cudaMemcpyAsync(f_dev + mv, moved_to, (size_t)mv * 8, cudaMemcpyHostToDevice, ctx->stream));
    MoveParams mp;
    for (int i = 0; i < nc; ++i) {
      mp.col[i] = static_cast<uint8_t*>(*col[i].ptr);
      mp.row_bytes[i] = col[i].row_bytes;
    }
    mp.n_cols = nc;
    mp.from = f_dev;
    mp.to = f_dev + mv;
    mp.n_moves = mv;
    dense_move_rows_kernel<<<(unsigned)((mv + 7) / 8), 256, 0, ctx->stream>>>(mp);
    SB_CUDA(cudaGetLastError());
  }
  // the vacated tail [keep, n) returns to the fill of unused capacity
  for (int i = 0; i < nc; ++i)
    SB_CUDA(cudaMemsetAsync(static_cast<uint8_t*>(*col[i].ptr) + (size_t)keep * col[i].row_bytes, col[i].fill,
                            (size_t)n * col[i].row_bytes, ctx->stream));
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  ix.n = keep;
  ix.n_pad = round_rows(keep);
  return SB_OK;
}

int sb_dense_set_mode(sb_ctx* ctx, int mode) {
  SB_REQUIRE(ctx != nullptr && mode >= 0 && mode <= 2, SB_ERR_ARG, "sb_dense_set_mode: bad arguments");
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->dense_mode = mode;
  return SB_OK;
}

int64_t sb_dense_count(sb_ctx* ctx, int slot) {
  if (!ctx || slot < 0 || slot >= SB_MAX_DENSE_SLOTS) return -1;
  return ctx->dense[slot].n;
}

int32_t sb_dense_dim(sb_ctx* ctx, int slot) {
  if (!ctx || slot < 0 || slot >= SB_MAX_DENSE_SLOTS) return -1;
  return ctx->dense[slot].d;
}

int sb_dense_topk_dev(sb_ctx* ctx, int slot, const float* q_dev, int32_t B, int32_t k, int64_t* out_ids_dev,
                      double* out_scores_dev, int32_t* out_counts_dev, void* stream) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_topk_dev: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_topk_dev: bad slot %d", slot);
  SB_REQUIRE(B >= 0 && k > 0, SB_ERR_ARG, "sb_dense_topk_dev: bad B=%d k=%d", B, k);
  if (B == 0) return SB_OK;
  SB_REQUIRE(q_dev && out_ids_dev && out_scores_dev && out_counts_dev, SB_ERR_ARG, "sb_dense_topk_dev: NULL buffer");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = pick_stream(ctx, stream);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_topk: dense slot %d has no index loaded", slot);
  if (ix.n == 0) {
    fill_empty_topk_kernel<<<(B * k + 255) / 256, 256, 0, st>>>(out_ids_dev, out_scores_dev, out_counts_dev, B, k);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
  }
  float* q_pad = nullptr;
  int rc = sb_dense_pad_queries(ctx, ix, q_dev, B, true, &q_pad, st);
  if (rc) return rc;
  return dense_topk_enqueue(ctx, ix, q_pad, B, k, out_ids_dev, out_scores_dev, out_counts_dev, st);
}

int sb_dense_topk(sb_ctx* ctx, int slot, const float* q, int32_t B, int32_t k, int64_t* out_ids, double* out_scores,
                  int32_t* out_counts) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_topk: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_topk: bad slot %d", slot);
  SB_REQUIRE(B >= 0 && k > 0, SB_ERR_ARG, "sb_dense_topk: bad B=%d k=%d", B, k);
  if (B == 0) return SB_OK;
  SB_REQUIRE(q && out_ids && out_scores && out_counts, SB_ERR_ARG, "sb_dense_topk: NULL buffer");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = ctx->stream;
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_topk: dense slot %d has no index loaded", slot);
  if (ix.n == 0) {
    for (int i = 0; i < B * k; ++i) { out_ids[i] = -1; out_scores[i] = 0.0; }
    for (int i = 0; i < B; ++i) out_counts[i] = 0;
    return SB_OK;
  }
  int rc;
  const size_t qbytes = (size_t)B * ix.d * sizeof(float);
  const size_t nid = (size_t)B * k;
  // page-locked caller buffers are used in place; pageable ones go through the context's pinned staging
  const bool in_pinned = host_ptr_is_pinned(q);
  const bool out_pinned = host_ptr_is_pinned(out_ids) && host_ptr_is_pinned(out_scores) && host_ptr_is_pinned(out_counts);
  const float* q_src = q;
  if (!in_pinned) {
    if ((rc = ctx->pin_in.reserve(qbytes))) return rc;
    memcpy(ctx->pin_in.p, q, qbytes);
    q_src = ctx->pin_in.as<float>();
  }
  float* q_pad = nullptr;
  if ((rc = sb_dense_pad_queries(ctx, ix, q_src, B, false, &q_pad, st))) return rc;
  if ((rc = ctx->out_ids_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_sc_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_cnt_dev.reserve((size_t)B * 4))) return rc;
  if ((rc = dense_topk_enqueue(ctx, ix, q_pad, B, k, ctx->out_ids_dev.as<int64_t>(), ctx->out_sc_dev.as<double>(),
                               ctx->out_cnt_dev.as<int32_t>(), st)))
    return rc;
  if (out_pinned) {
    SB_CUDA(cudaMemcpyAsync(out_ids, ctx->out_ids_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(out_scores, ctx->out_sc_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(out_counts, ctx->out_cnt_dev.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    return SB_OK;
  }
  if ((rc = ctx->pin_out.reserve(nid * 16 + (size_t)B * 4))) return rc;
  uint8_t* po = ctx->pin_out.as<uint8_t>();
  SB_CUDA(cudaMemcpyAsync(po, ctx->out_ids_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(po + nid * 8, ctx->out_sc_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(po + nid * 16, ctx->out_cnt_dev.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  memcpy(out_ids, po, nid * 8);
  memcpy(out_scores, po + nid * 8, nid * 8);
  memcpy(out_counts, po + nid * 16, (size_t)B * 4);
  return SB_OK;
}

int sb_dense_fetch(sb_ctx* ctx, int slot, const int64_t* ids, int32_t n_ids, float* out) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_fetch: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_fetch: bad slot %d", slot);
  if (n_ids <= 0) return SB_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  const DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0 && ix.n > 0, SB_ERR_STATE, "sb_dense_fetch: dense slot %d is empty", slot);
  int rc;
  if ((rc = ctx->misc2_dev.reserve((size_t)n_ids * 8))) return rc;
  if ((rc = ctx->misc3_dev.reserve((size_t)n_ids * ix.d * 4))) return rc;
  SB_CUDA(cudaMemcpyAsync(ctx->misc2_dev.p, ids, (size_t)n_ids * 8, cudaMemcpyHostToDevice, ctx->stream));
  if (ix.storage == SB_STORAGE_U8)
    dense_fetch_u8_kernel<<<n_ids, 128, 0, ctx->stream>>>(ix.rows8, ix.d, ix.d_pad, ix.n, ix.id_base,
                                                          ctx->misc2_dev.as<int64_t>(), n_ids, ctx->misc3_dev.as<float>());
  else if (ix.storage == SB_STORAGE_F32)
    dense_fetch_f32_kernel<<<n_ids, 128, 0, ctx->stream>>>(ix.rows32, ix.metric == SB_METRIC_COSINE, ix.d, ix.d_pad, ix.n,
                                                           ix.id_base, ctx->misc2_dev.as<int64_t>(), n_ids,
                                                           ctx->misc3_dev.as<float>());
  else
    dense_fetch_kernel<<<n_ids, 128, 0, ctx->stream>>>(ix.rows, ix.cfac, ix.d, ix.d_pad, ix.n, ix.id_base,
                                                       ctx->misc2_dev.as<int64_t>(), n_ids, ctx->misc3_dev.as<float>());
  SB_CUDA(cudaGetLastError());
  SB_CUDA(cudaMemcpyAsync(out, ctx->misc3_dev.p, (size_t)n_ids * ix.d * 4, cudaMemcpyDeviceToHost, ctx->stream));
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  return SB_OK;
}

int sb_dense_tags_load(sb_ctx* ctx, int slot, int32_t field, const int32_t* codes, int64_t n) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_tags_load: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_tags_load: bad slot %d", slot);
  SB_REQUIRE(field >= 0 && field < SB_MAX_TAG_FIELDS, SB_ERR_ARG, "sb_dense_tags_load: field %d out of range [0,%d)",
             field, SB_MAX_TAG_FIELDS);
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_tags_load: dense slot %d has no index loaded", slot);
  SB_REQUIRE(n == ix.n, SB_ERR_ARG, "sb_dense_tags_load: %lld codes for %lld rows", (long long)n, (long long)ix.n);
  SB_REQUIRE(n == 0 || codes != nullptr, SB_ERR_ARG, "sb_dense_tags_load: codes is NULL");
  for (int64_t i = 0; i < n; ++i)
    SB_REQUIRE(codes[i] >= -1, SB_ERR_ARG, "sb_dense_tags_load: code %d at row %lld (must be >= -1)", codes[i],
               (long long)i);
  return dense_payload_load(ctx, ix, tag_column(ix, field), codes, n);
}

int sb_dense_topk_filtered_dev(sb_ctx* ctx, int slot, const float* q_dev, int32_t B, int32_t k,
                               const int32_t* f_off_dev, int32_t n_conds, const int32_t* f_field_dev,
                               const int32_t* f_code_dev, int64_t* out_ids_dev, double* out_scores_dev,
                               int32_t* out_counts_dev, void* stream) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_topk_filtered_dev: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_topk_filtered_dev: bad slot %d", slot);
  SB_REQUIRE(B >= 0 && k > 0 && n_conds >= 0, SB_ERR_ARG, "sb_dense_topk_filtered_dev: bad B=%d k=%d n_conds=%d", B, k,
             n_conds);
  if (B == 0) return SB_OK;
  SB_REQUIRE(q_dev && f_off_dev && out_ids_dev && out_scores_dev && out_counts_dev, SB_ERR_ARG,
             "sb_dense_topk_filtered_dev: NULL buffer");
  SB_REQUIRE(n_conds == 0 || (f_field_dev && f_code_dev), SB_ERR_ARG, "sb_dense_topk_filtered_dev: NULL conditions");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = pick_stream(ctx, stream);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_topk_filtered_dev: dense slot %d has no index loaded", slot);
  // the conditions decide which kernels run: read them once
  std::vector<int32_t> h((size_t)B + 1 + 2 * (size_t)n_conds);
  SB_CUDA(cudaMemcpyAsync(h.data(), f_off_dev, (size_t)(B + 1) * 4, cudaMemcpyDeviceToHost, st));
  if (n_conds) {
    SB_CUDA(cudaMemcpyAsync(h.data() + B + 1, f_field_dev, (size_t)n_conds * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaMemcpyAsync(h.data() + B + 1 + n_conds, f_code_dev, (size_t)n_conds * 4, cudaMemcpyDeviceToHost, st));
  }
  SB_CUDA(cudaStreamSynchronize(st));
  SB_REQUIRE(h[B] == n_conds, SB_ERR_ARG, "sb_dense_topk_filtered_dev: f_off[B] = %d != n_conds = %d", h[B], n_conds);
  if (ix.n == 0) {
    fill_empty_topk_kernel<<<(B * k + 255) / 256, 256, 0, st>>>(out_ids_dev, out_scores_dev, out_counts_dev, B, k);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
  }
  float* q_pad = nullptr;
  int rc = sb_dense_pad_queries(ctx, ix, q_dev, B, true, &q_pad, st);
  if (rc) return rc;
  return dense_topk_filtered_enqueue(ctx, ix, q_pad, B, k, h.data(), h.data() + B + 1, h.data() + B + 1 + n_conds,
                                     out_ids_dev, out_scores_dev, out_counts_dev, st);
}

int sb_dense_topk_filtered(sb_ctx* ctx, int slot, const float* q, int32_t B, int32_t k, const int32_t* f_off,
                           const int32_t* f_field, const int32_t* f_code, int64_t* out_ids, double* out_scores,
                           int32_t* out_counts) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_topk_filtered: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_topk_filtered: bad slot %d", slot);
  SB_REQUIRE(B >= 0 && k > 0, SB_ERR_ARG, "sb_dense_topk_filtered: bad B=%d k=%d", B, k);
  if (B == 0) return SB_OK;
  SB_REQUIRE(q && f_off && out_ids && out_scores && out_counts, SB_ERR_ARG, "sb_dense_topk_filtered: NULL buffer");
  SB_REQUIRE(f_off[B] == 0 || (f_field && f_code), SB_ERR_ARG, "sb_dense_topk_filtered: NULL conditions");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = ctx->stream;
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_topk_filtered: dense slot %d has no index loaded", slot);
  if (ix.n == 0) {
    for (int i = 0; i < B * k; ++i) { out_ids[i] = -1; out_scores[i] = 0.0; }
    for (int i = 0; i < B; ++i) out_counts[i] = 0;
    return SB_OK;
  }
  int rc;
  const size_t qbytes = (size_t)B * ix.d * sizeof(float);
  const size_t nid = (size_t)B * k;
  if ((rc = ctx->pin_in.reserve(qbytes))) return rc;
  SB_CUDA(cudaStreamSynchronize(st));
  memcpy(ctx->pin_in.p, q, qbytes);
  float* q_pad = nullptr;
  if ((rc = sb_dense_pad_queries(ctx, ix, ctx->pin_in.as<float>(), B, false, &q_pad, st))) return rc;
  if ((rc = ctx->out_ids_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_sc_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_cnt_dev.reserve((size_t)B * 4))) return rc;
  if ((rc = dense_topk_filtered_enqueue(ctx, ix, q_pad, B, k, f_off, f_field, f_code, ctx->out_ids_dev.as<int64_t>(),
                                        ctx->out_sc_dev.as<double>(), ctx->out_cnt_dev.as<int32_t>(), st)))
    return rc;
  SB_CUDA(cudaMemcpyAsync(out_ids, ctx->out_ids_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_scores, ctx->out_sc_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_counts, ctx->out_cnt_dev.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return SB_OK;
}

int sb_dense_values_load(sb_ctx* ctx, int slot, int32_t field, const double* vals, int64_t n) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_values_load: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_values_load: bad slot %d", slot);
  SB_REQUIRE(field >= 0 && field < SB_MAX_VALUE_FIELDS, SB_ERR_ARG,
             "sb_dense_values_load: field %d out of range [0,%d)", field, SB_MAX_VALUE_FIELDS);
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_values_load: dense slot %d has no index loaded", slot);
  SB_REQUIRE(n == ix.n, SB_ERR_ARG, "sb_dense_values_load: %lld values for %lld rows", (long long)n, (long long)ix.n);
  SB_REQUIRE(n == 0 || vals != nullptr, SB_ERR_ARG, "sb_dense_values_load: vals is NULL");
  return dense_payload_load(ctx, ix, value_column(ix, field), vals, n);
}

int sb_dense_values_write(sb_ctx* ctx, int slot, int32_t field, const int64_t* rows, const double* vals, int64_t n) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_values_write: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_values_write: bad slot %d", slot);
  SB_REQUIRE(field >= 0 && field < SB_MAX_VALUE_FIELDS, SB_ERR_ARG,
             "sb_dense_values_write: field %d out of range [0,%d)", field, SB_MAX_VALUE_FIELDS);
  SB_REQUIRE(n >= 0, SB_ERR_ARG, "sb_dense_values_write: bad n=%lld", (long long)n);
  SB_REQUIRE(n == 0 || (rows != nullptr && vals != nullptr), SB_ERR_ARG, "sb_dense_values_write: NULL buffer");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_values_write: dense slot %d has no index loaded", slot);
  SB_REQUIRE(ix.vals[field] != nullptr, SB_ERR_STATE, "sb_dense_values_write: field %d has no value column loaded",
             field);
  std::vector<int64_t> sorted;
  int rc = check_rows("sb_dense_values_write", rows, n, ix.n, sorted);
  if (rc) return rc;
  if (n == 0) return SB_OK;
  SB_CUDA(cudaDeviceSynchronize());
  if ((rc = ctx->misc2_dev.reserve((size_t)n * 16))) return rc;
  int64_t* r_dev = ctx->misc2_dev.as<int64_t>();
  double* v_dev = reinterpret_cast<double*>(r_dev + n);
  SB_CUDA(cudaMemcpyAsync(r_dev, rows, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  SB_CUDA(cudaMemcpyAsync(v_dev, vals, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  dense_values_scatter_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(ix.vals[field], r_dev, v_dev, n);
  SB_CUDA(cudaGetLastError());
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  return SB_OK;
}

int sb_dense_topk_where(sb_ctx* ctx, int slot, const float* q, int32_t B, int32_t k, const int32_t* p_off,
                        const sb_pred* prog, const int32_t* pool, int32_t n_pool, int64_t* out_ids, double* out_scores,
                        int32_t* out_counts) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_topk_where: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_topk_where: bad slot %d", slot);
  SB_REQUIRE(B >= 0 && k > 0, SB_ERR_ARG, "sb_dense_topk_where: bad B=%d k=%d", B, k);
  if (B == 0) return SB_OK;
  SB_REQUIRE(q && p_off && out_ids && out_scores && out_counts, SB_ERR_ARG, "sb_dense_topk_where: NULL buffer");
  SB_REQUIRE(p_off[B] == 0 || prog != nullptr, SB_ERR_ARG, "sb_dense_topk_where: NULL program");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = ctx->stream;
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_topk_where: dense slot %d has no index loaded", slot);
  int rc = where_validate("sb_dense_topk_where", ix, B, p_off, prog, pool, n_pool);
  if (rc) return rc;
  SB_REQUIRE(k <= kDenseMaxK, SB_ERR_UNSUPPORTED, "dense: top_k %d too large (max %d per call)", k, kDenseMaxK);
  if (ix.n == 0) {
    for (int i = 0; i < B * k; ++i) { out_ids[i] = -1; out_scores[i] = 0.0; }
    for (int i = 0; i < B; ++i) out_counts[i] = 0;
    return SB_OK;
  }
  const size_t qbytes = (size_t)B * ix.d * sizeof(float);
  const size_t nid = (size_t)B * k;
  if ((rc = ctx->pin_in.reserve(qbytes))) return rc;
  SB_CUDA(cudaStreamSynchronize(st));
  memcpy(ctx->pin_in.p, q, qbytes);
  float* q_pad = nullptr;
  if ((rc = sb_dense_pad_queries(ctx, ix, ctx->pin_in.as<float>(), B, false, &q_pad, st))) return rc;
  if ((rc = ctx->out_ids_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_sc_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_cnt_dev.reserve((size_t)B * 4))) return rc;
  if ((rc = dense_topk_where_enqueue(ctx, ix, q_pad, B, k, p_off, prog, pool, ctx->out_ids_dev.as<int64_t>(),
                                     ctx->out_sc_dev.as<double>(), ctx->out_cnt_dev.as<int32_t>(), st)))
    return rc;
  SB_CUDA(cudaMemcpyAsync(out_ids, ctx->out_ids_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_scores, ctx->out_sc_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_counts, ctx->out_cnt_dev.p, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return SB_OK;
}

int sb_dense_recommend(sb_ctx* ctx, int slot, const float* ex, int32_t m, const int32_t* r_off, const int32_t* n_pos,
                       const int32_t* strategy, int32_t R, int32_t k, const int32_t* p_off, const sb_pred* prog,
                       const int32_t* pool, int32_t n_pool, int64_t* out_ids, double* out_scores, int32_t* out_counts) {
  const char* who = "sb_dense_recommend";
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "%s: ctx is NULL", who);
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "%s: bad slot %d", who, slot);
  SB_REQUIRE(R >= 0 && m >= 0 && k > 0, SB_ERR_ARG, "%s: bad R=%d m=%d k=%d", who, R, m, k);
  SB_REQUIRE(k <= kDenseMaxK, SB_ERR_UNSUPPORTED, "%s: top_k %d too large (max %d per call)", who, k, kDenseMaxK);
  if (R == 0) return SB_OK;
  SB_REQUIRE(ex && r_off && n_pos && strategy && out_ids && out_scores && out_counts, SB_ERR_ARG, "%s: NULL buffer", who);
  SB_REQUIRE(r_off[0] == 0 && r_off[R] == m, SB_ERR_ARG, "%s: r_off must run from 0 to m = %d", who, m);
  std::vector<RecoReq> req((size_t)R);
  for (int r = 0; r < R; ++r) {
    const int32_t mr = r_off[r + 1] - r_off[r];
    SB_REQUIRE(mr >= 1 && mr <= SB_RECO_MAX_EXAMPLES, SB_ERR_ARG, "%s: request %d has %d examples (1 to %d)", who, r, mr,
               SB_RECO_MAX_EXAMPLES);
    SB_REQUIRE(n_pos[r] >= 0 && n_pos[r] <= mr, SB_ERR_ARG, "%s: request %d: n_pos %d outside [0, %d]", who, r, n_pos[r],
               mr);
    SB_REQUIRE(strategy[r] == SB_RECO_BEST_SCORE || strategy[r] == SB_RECO_SUM_SCORES, SB_ERR_ARG,
               "%s: request %d: strategy %d", who, r, strategy[r]);
    req[(size_t)r] = {r_off[r], mr, n_pos[r], strategy[r]};
  }
  SB_REQUIRE(p_off == nullptr || p_off[R] == 0 || prog != nullptr, SB_ERR_ARG, "%s: NULL program", who);
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = ctx->stream;
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "%s: dense slot %d has no index loaded", who, slot);
  SB_REQUIRE(ix.metric != SB_METRIC_EUCLID, SB_ERR_UNSUPPORTED, "%s: best_score / sum_scores on a Euclid slot", who);
  for (int64_t i = 0; i < (int64_t)m * ix.d; ++i)
    SB_REQUIRE(std::isfinite(ex[i]), SB_ERR_ARG, "%s: example %lld has a NaN or infinite value", who,
               (long long)(i / ix.d));
  int rc;
  if (p_off && (rc = where_validate(who, ix, R, p_off, prog, pool, n_pool))) return rc;
  if (ix.n == 0) {
    for (int64_t i = 0; i < (int64_t)R * k; ++i) { out_ids[i] = -1; out_scores[i] = 0.0; }
    for (int i = 0; i < R; ++i) out_counts[i] = 0;
    return SB_OK;
  }
  const size_t nid = (size_t)R * k;
  if ((rc = ctx->pin_in.reserve((size_t)m * ix.d * sizeof(float)))) return rc;
  SB_CUDA(cudaStreamSynchronize(st));
  memcpy(ctx->pin_in.p, ex, (size_t)m * ix.d * sizeof(float));
  float* ex_pad = nullptr;
  if ((rc = sb_dense_pad_queries(ctx, ix, ctx->pin_in.as<float>(), m, false, &ex_pad, st))) return rc;
  if ((rc = ctx->out_ids_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_sc_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_cnt_dev.reserve((size_t)R * 4))) return rc;
  if ((rc = dense_reco_enqueue(ctx, ix, ex_pad, m, req.data(), R, k, p_off && p_off[R] > 0 ? p_off : nullptr, prog, pool,
                               ctx->out_ids_dev.as<int64_t>(), ctx->out_sc_dev.as<double>(),
                               ctx->out_cnt_dev.as<int32_t>(), st)))
    return rc;
  SB_CUDA(cudaMemcpyAsync(out_ids, ctx->out_ids_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_scores, ctx->out_sc_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_counts, ctx->out_cnt_dev.p, (size_t)R * 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return SB_OK;
}

int sb_dense_groups(sb_ctx* ctx, int slot, const float* q, int32_t B, int32_t group_field, int32_t L, int32_t G,
                    const int32_t* f_off, const int32_t* f_field, const int32_t* f_code, int32_t* out_group_code,
                    int32_t* out_group_hits, int64_t* out_ids, double* out_scores, int32_t* out_n_groups) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_dense_groups: ctx is NULL");
  SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_dense_groups: bad slot %d", slot);
  SB_REQUIRE(B >= 0, SB_ERR_ARG, "sb_dense_groups: bad B=%d", B);
  SB_REQUIRE(L >= 1 && L <= kDenseMaxK && G >= 1 && G <= kDenseMaxK, SB_ERR_ARG,
             "sb_dense_groups: limit %d and group_size %d must be in [1, %d]", L, G, kDenseMaxK);
  SB_REQUIRE(group_field >= 0 && group_field < SB_MAX_TAG_FIELDS, SB_ERR_ARG,
             "sb_dense_groups: group field %d out of range [0,%d)", group_field, SB_MAX_TAG_FIELDS);
  if (B == 0) return SB_OK;
  SB_REQUIRE(q && out_group_code && out_group_hits && out_ids && out_scores && out_n_groups, SB_ERR_ARG,
             "sb_dense_groups: NULL buffer");
  int n_conds = 0;
  if (f_off) {
    SB_REQUIRE(f_off[0] == 0, SB_ERR_ARG, "sb_dense_groups: f_off[0] must be 0");
    for (int b = 0; b < B; ++b)
      SB_REQUIRE(f_off[b + 1] >= f_off[b], SB_ERR_ARG, "sb_dense_groups: f_off is not non-decreasing at %d", b);
    n_conds = f_off[B];
    SB_REQUIRE(n_conds == 0 || (f_field && f_code), SB_ERR_ARG, "sb_dense_groups: NULL conditions");
    for (int i = 0; i < n_conds; ++i)
      SB_REQUIRE(f_field[i] >= 0 && f_field[i] < SB_MAX_TAG_FIELDS, SB_ERR_ARG, "sb_dense_groups: field %d out of range",
                 f_field[i]);
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = ctx->stream;
  DenseIndex& ix = ctx->dense[slot];
  SB_REQUIRE(ix.d > 0, SB_ERR_STATE, "sb_dense_groups: dense slot %d has no index loaded", slot);
  SB_REQUIRE(ix.tags[group_field] != nullptr, SB_ERR_STATE, "sb_dense_groups: field %d has no tag column loaded",
             group_field);
  for (int i = 0; i < n_conds; ++i)
    SB_REQUIRE(ix.tags[f_field[i]] != nullptr, SB_ERR_STATE, "sb_dense_groups: field %d has no tag column loaded",
               f_field[i]);
  const size_t BL = (size_t)B * L, BLG = BL * G;
  if (ix.n == 0) {
    for (int b = 0; b < B; ++b) out_n_groups[b] = 0;
    for (size_t i = 0; i < BL; ++i) { out_group_code[i] = -1; out_group_hits[i] = 0; }
    for (size_t i = 0; i < BLG; ++i) { out_ids[i] = -1; out_scores[i] = 0.0; }
    return SB_OK;
  }
  int rc;
  const size_t qbytes = (size_t)B * ix.d * sizeof(float);
  if ((rc = ctx->pin_in.reserve(qbytes))) return rc;
  SB_CUDA(cudaStreamSynchronize(st));
  memcpy(ctx->pin_in.p, q, qbytes);
  float* q_pad = nullptr;
  if ((rc = sb_dense_pad_queries(ctx, ix, ctx->pin_in.as<float>(), B, false, &q_pad, st))) return rc;
  GroupLayout o;
  if ((rc = dense_groups_enqueue(ctx, ix, q_pad, B, group_field, L, G, f_off, f_field, f_code, &o, st))) return rc;
  const uint8_t* res = ctx->grp_res_dev.as<uint8_t>();
  SB_CUDA(cudaMemcpyAsync(out_n_groups, res + o.n_groups, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_group_code, res + o.g_code, BL * 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_group_hits, res + o.g_hits, BL * 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_ids, res + o.h_ids, BLG * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(out_scores, res + o.h_scores, BLG * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return SB_OK;
}

int sb_dense_group_rounds(sb_ctx* ctx, int64_t* hist, int32_t n) {
  SB_REQUIRE(ctx != nullptr && n >= 0 && (n == 0 || hist != nullptr), SB_ERR_ARG, "sb_dense_group_rounds: bad arguments");
  std::lock_guard<std::mutex> lk(ctx->mu);
  for (int i = 0; i < n; ++i) hist[i] = 0;
  for (size_t r = 0; r < ctx->grp_rounds.size() && n > 0; ++r) hist[std::min<size_t>(r, (size_t)n - 1)] += ctx->grp_rounds[r];
  return SB_OK;
}

int64_t sb_dense_fallback_count(sb_ctx* ctx) {
  if (!ctx) return -1;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  if (ctx->fb_count_dev.cap == 0) return 0;
  unsigned long long v = 0;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpy(&v, ctx->fb_count_dev.p, 8, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return (int64_t)v;
}

}  // extern "C"
