// dense_mma.cu -- K1b: batched-query dense scan on the Hopper tensor cores (wgmma / TMA), sm_90a.
//
// One HBM pass over the fp16 corpus serves a whole GROUP of up to 256 queries: the scores of a 128-row corpus tile
// against all queries of the group are one accumulator  D[128, N] = A[128, D] * Q[N, D]^T  (A = corpus tile, B = the
// normalised fp16 query block, both K-major fp16 streamed by TMA in 64-column SWIZZLE_128B boxes; D in the registers of
// two consumer warpgroups, 64 corpus rows each).
//   * dense_scan_mma_kernel<QBN>   N = QBN = 16 / 32 / 64 / 128 / 256 queries (m64nQBNk16).
// A ring stage holds one corpus box (16 KB) and the matching box of the query block (QBN x 128 B), so shared memory does
// not grow with d: at QBN = 256 four 48 KB stages fit the 227 KB a block may use.
// At QBN = 256 a 16 KB corpus box feeds 8 MMAs of 64 x 256 x 16.
//
// Every CTA loads the query boxes itself (512 KB per tile from L2 at d = 1024).  Those L2 reads do not bound the pass,
// and sharing them across a 2-CTA cluster by TMA multicast measured no faster on the H100.  The serial epilogue does
// bound it: skipping it takes a 256-query pass from 1.07 to 0.79 ms (DESIGN.md K1b).  So the epilogue keeps global loads
// off its critical path: a tile's row scales are loaded before its MMAs, and the thresholds once per column pair.  It
// also tests every score without a branch, into one pass bit per accumulator register, and walks only the set bits.
//
// Exactness (dense_common.cuh, DESIGN.md "K1: exactness"):
//   * queries are L2-normalised before the fp16 rounding (cosine is scale invariant; the caller's scale never reaches
//     the fp16 range) and eps[q] = ||fp16(qn) - qn|| + accumulation bound is computed per query;
//   * a sampling pass gives every query a SAFE threshold: (k-th best approximate score of a corpus sample) - 2 eps is
//     <= (global k-th best) - 2 eps, the lower edge of the hand-off window, so every window member survives the epilogue;
//   * survivors are appended to per-(CTA, query) lists; a list that overflows its capacity raises the query's fallback
//     flag instead of dropping anything silently;
//   * dense_select_kernel finds the k-th best approximate key (radix select), gathers EVERY survivor inside the window
//     below it and re-scores them all in fp64 against the stored rows and the caller's fp32 query; a window larger than
//     the winner buffer raises the fallback flag (dense_exact_fallback_kernel, dense.cu).
//
// Warp roles (288 threads, 1 CTA / SM, persistent): warps 0..7 = two consumer warpgroups (MMA + epilogue; a thread holds
// two corpus rows x QBN / 4 query columns of the accumulator), warp 8 = TMA producer.
//
// Uint8 storage (ST = SB_STORAGE_U8, DESIGN.md K1i): the corpus box is 64 bytes x 128 rows (8 KB, no swizzle) of the
// integer rows x.  Each consumer thread reads 16 bytes of its two accumulator rows per box, turns them into f16x2 A
// fragments in registers (exact: 0..255 are fp16 integers) and issues the register-A form of the same MMAs.  The query
// block's columns are permuted inside each 64-column block to match (u8_query_column).  Every other step is the same.
#include <cuda.h>

#include <math.h>

#include <algorithm>
#include <vector>

#include "dense_common.cuh"
#include "dense_mma.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kTileRows = 128;
constexpr int kBK = 64;                       // fp16 elements per 128-byte swizzle row
constexpr uint32_t kATileBytes = kTileRows * kBK * 2;   // 16 KB
constexpr uint32_t kATileBytesU8 = kTileRows * kBK;     // 8 KB: a uint8 corpus box
constexpr int kConsumerWarps = 8;
constexpr int kMmaThreads = 32 * kConsumerWarps + 32;
constexpr int kQbnMax = 256;                  // queries per group (m64n256k16)
constexpr int kSampleRows = 16;               // corpus rows behind one sampling-pass key (one warp's accumulator rows)
constexpr int kSampleKeys = kTileRows / kSampleRows;   // sampling-pass keys per (tile, query)
constexpr int kSelectThreads = 512;
constexpr int kSelStage = 8192;               // survivors staged in shared memory by dense_select_kernel (64 KB)
constexpr int kSelTop = 2048;                 // window (winner) buffer; larger windows go to the exact fallback

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar,
                                            uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], "
      "[%4], %5;" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(bar), "l"(policy)
      : "memory");
}
// 4 bytes b0..b3 -> the f16x2 pair (b0, b1) (sel 0x5140) or (b2, b3) (sel 0x7362): 1024 + b has the bit pattern
// 0x6400 | b, and subtracting 1024 is exact
__device__ __forceinline__ uint32_t u8_f16x2(uint32_t w, uint32_t sel) {
  const uint32_t h = __byte_perm(w, 0x64646464u, sel);
  uint32_t r;
  asm("sub.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(h), "r"(0x64006400u));
  return r;
}

// L2 prefetch of a tensor-map box (no shared-memory destination): keeps more HBM requests in flight than the ring holds
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* map, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(map), "r"(c0), "r"(c1) : "memory");
}

// *ptr if `live`, else 0, through the read-only path.  volatile: the load is issued where it is written (ahead of a
// tile's MMAs) instead of being moved to its first use.
__device__ __forceinline__ float ldg_early(const float* ptr, bool live) {
  float v = 0.f;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.u32 p, %2, 0;\n"
      "@p ld.global.nc.f32 %0, [%1];\n"
      "}\n"
      : "+f"(v)
      : "l"(ptr), "r"((uint32_t)live));
  return v;
}

// acc[32 w + b] for a bit index b known only at run time: a tree of selects on the bits of b over the word's values.
// Indexing the register array with b would move the accumulator to local memory, and a switch would branch apart the
// lanes of a warp.  w must be a constant once the caller's loop is unrolled.
template <int N>
__device__ __forceinline__ float acc_word_at(const float (&acc)[N], int w, int b) {
  constexpr int kN = N < 32 ? N : 32;   // accumulator values behind one mask word
  float v[kN];
#pragma unroll
  for (int i = 0; i < kN; ++i) v[i] = acc[32 * w + i];
#pragma unroll
  for (int s = 1; s < kN; s <<= 1)
#pragma unroll
    for (int i = 0; i < kN; i += 2 * s) v[i] = (b & s) ? v[i + s] : v[i];
  return v[0];
}

struct MmaScanParams {
  const float* inv_norm;
  const float* thr_init;        // [QBN] safe initial thresholds (NULL = -inf: sampling pass)
  unsigned long long* cand;     // [QBN][grid][capg]
  int32_t* counts;              // [QBN][grid]
  int32_t* fallback;            // [QBN] raised when a (CTA, query) list overflows capg (NULL: cannot overflow)
  int64_t n;                    // valid rows
  int32_t kb_count;             // d_pad / 64
  int32_t num_tiles;            // tiles visited by this launch
  int32_t tile_first, tile_step; // global tile index = tile_first + t * tile_step,  t in [0, num_tiles)
  int32_t capg;
  int32_t stages;
  int32_t prefetch;             // boxes (16 KB) prefetched into L2 beyond the shared-memory ring (0 = off)
  const uint32_t* mask;         // FILTER only: match bits of the group's queries, mask[(row / 32) * mask_qs + column]
  int32_t mask_qs;
  const float* hh;              // EUCLID only: per-row h (>= ||v||^2 / 2)
  const float* rq;              // EUCLID only: [QBN] (float)||q|| of the group's queries
};
// STORE mode reads the same parameters (keeping every other instantiation's code unchanged): cand is the float key
// buffer, keys[col * capg + row], and mask_qs the number of columns stored.

// Key of a row (dense.cu dense_scan_kernel): acc * scale[row], EUCLID r * (acc * scale[row]) - h[row].
// STORE (recommendation, DESIGN.md K1j): no threshold and no lists; every live row's key of every column < mask_qs is
// written to the key buffer (MmaScanParams).
template <int QBN, bool FILTER, bool EUCLID, int ST, bool STORE = false>
__global__ void __launch_bounds__(kMmaThreads, 1)
dense_scan_mma_kernel(const __grid_constant__ CUtensorMap tm_rows, const __grid_constant__ CUtensorMap tm_q,
                      const MmaScanParams p) {
  extern __shared__ uint8_t msm_raw[];
  const uint32_t raw = smem_u32(msm_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;  // SWIZZLE_128B operands need 1024-byte alignment
  uint8_t* sm = msm_raw + (base - raw);
  constexpr bool U8 = ST == SB_STORAGE_U8;
  constexpr uint32_t kABytes = U8 ? kATileBytesU8 : kATileBytes;   // one corpus box
  constexpr uint32_t kQBoxBytes = QBN * kBK * 2;              // one 64-column box of the query block
  constexpr uint32_t kStageBytes = kABytes + kQBoxBytes;      // corpus box, then query box
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + (size_t)p.stages * kStageBytes);
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + p.stages);
  float* thr = reinterpret_cast<float*>(bars + 2 * p.stages);   // [QBN], 8-byte aligned
  const uint32_t thr_s = smem_u32(thr);                         // read-only once the block has synchronised
  int* cnt = reinterpret_cast<int*>(thr + QBN);                 // [QBN]
  float* rq_s = reinterpret_cast<float*>(cnt + QBN);                             // [QBN] EUCLID only

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grid = gridDim.x, cta = blockIdx.x;
  const int my_tiles = cta < p.num_tiles ? (p.num_tiles - 1 - cta) / grid + 1 : 0;
  auto tile_row = [&](int t) { return (p.tile_first + (cta + t * grid) * p.tile_step) * kTileRows; };

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, kConsumerWarps);   // one arrival per consumer warp
    }
    mbar_fence_init();
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_rows) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_q) : "memory");
  }
  for (int i = threadIdx.x; i < QBN; i += blockDim.x) {
    thr[i] = p.thr_init ? p.thr_init[i] : -INFINITY;
    cnt[i] = 0;
    if constexpr (EUCLID) rq_s[i] = p.rq[i];
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ---------------------------------------------------------------- TMA producer
    if (lane == 0) {
      const uint64_t pol_corpus = policy_evict_first();   // 2 GB stream past the query block
      const uint64_t pol_query = policy_evict_last();     // read again by every tile
      int it = 0;
      const int total_it = my_tiles * p.kb_count;
      for (int t = 0; t < my_tiles; ++t) {
        const int row = tile_row(t);
        for (int kb = 0; kb < p.kb_count; ++kb, ++it) {
          const int s = it % p.stages;
          const uint32_t use = (uint32_t)(it / p.stages);
          const int pf = it + p.stages + p.prefetch;   // a box the ring will only reach later: pull it into L2 now
          if (p.prefetch > 0 && pf < total_it) {
            const int pt = pf / p.kb_count, pkb = pf - pt * p.kb_count;
            tma_prefetch_l2_2d(&tm_rows, pkb * kBK, tile_row(pt));
          }
          if (it >= p.stages) mbar_wait(bar_empty + 8 * s, (use & 1u) ^ 1u);
          const uint32_t stage = base + (uint32_t)s * kStageBytes;
          mbar_expect_tx(bar_full + 8 * s, kStageBytes);   // both boxes complete on the stage's one barrier
          tma_load_2d(stage, &tm_rows, kb * kBK, row, bar_full + 8 * s, pol_corpus);
          tma_load_2d(stage + kABytes, &tm_q, kb * kBK, 0, bar_full + 8 * s, pol_query);
        }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumer warpgroups: MMA + epilogue
    const int wg = warp >> 2;
    unsigned long long* my_cand = p.cand + (size_t)cta * p.capg;
    const size_t q_stride = (size_t)grid * p.capg;
    int it = 0;
    for (int t = 0; t < my_tiles; ++t) {
      // this thread's accumulator rows: row0 and row0 + 8; columns 8 j + 2 (lane % 4) + {0, 1}.  Their per-row scales are
      // loaded before the MMAs, so the epilogue does not start with a global-memory round trip.
      const int64_t row0 = (int64_t)tile_row(t) + wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const bool live0 = row0 < p.n, live1 = row0 + 8 < p.n;
      const float invn0 = ldg_early(p.inv_norm + row0, live0), invn1 = ldg_early(p.inv_norm + row0 + 8, live1);
      float h0 = 0.f, h1 = 0.f;
      if constexpr (EUCLID) {
        h0 = ldg_early(p.hh + row0, live0);
        h1 = ldg_early(p.hh + row0 + 8, live1);
      }
      float acc[QBN / 2];
      if constexpr (U8) {
        // this thread's 16 bytes of rows row0 and row0 + 8 in a box (64-byte rows): one warp reads 8 rows x 64
        // contiguous bytes per load.  A fragments of box kb stay live until its MMAs retire, one box after they are
        // issued, so the boxes alternate between two register sets.
        const uint32_t a_off = (uint32_t)(wg * 64 + (warp & 3) * 16 + (lane >> 2)) * (uint32_t)kBK + 16u * (lane & 3);
        uint32_t fa[16], fb[16];
        auto box = [&](int kb, uint32_t(&a)[16]) {
          const int s = it % p.stages;
          mbar_wait(bar_full + 8 * s, (uint32_t)(it / p.stages) & 1u);
          const uint32_t stage = base + (uint32_t)s * kStageBytes;
          uint32_t w0[4], w1[4];
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(w0[0]), "=r"(w0[1]), "=r"(w0[2]), "=r"(w0[3])
                       : "r"(stage + a_off));
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(w1[0]), "=r"(w1[1]), "=r"(w1[2]), "=r"(w1[3])
                       : "r"(stage + a_off + 8u * kBK));
#pragma unroll
          for (int k = 0; k < kBK / 16; ++k) {   // word k holds bytes 16 t + 4 k .. + 3: k16 step k
            a[4 * k + 0] = u8_f16x2(w0[k], 0x5140u);
            a[4 * k + 1] = u8_f16x2(w1[k], 0x5140u);
            a[4 * k + 2] = u8_f16x2(w0[k], 0x7362u);
            a[4 * k + 3] = u8_f16x2(w1[k], 0x7362u);
          }
          const uint64_t db = wgmma_desc_sw128(stage + kABytes);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBK / 16; ++k)
            WgmmaRA<QBN>::mma(acc, a[4 * k], a[4 * k + 1], a[4 * k + 2], a[4 * k + 3], db + (uint64_t)(2 * k),
                              (kb | k) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          __syncwarp();
          if (kb > 0 && lane == 0) mbar_arrive(bar_empty + 8 * ((it - 1) % p.stages));
          ++it;
        };
        for (int kb = 0; kb < p.kb_count; kb += 2) {
          box(kb, fa);
          if (kb + 1 < p.kb_count) box(kb + 1, fb);
        }
      } else {
        for (int kb = 0; kb < p.kb_count; ++kb, ++it) {
          const int s = it % p.stages;
          mbar_wait(bar_full + 8 * s, (uint32_t)(it / p.stages) & 1u);
          const uint32_t stage = base + (uint32_t)s * kStageBytes;
          const uint64_t da = wgmma_desc_sw128(stage + (uint32_t)wg * (kATileBytes / 2));
          const uint64_t db = wgmma_desc_sw128(stage + kATileBytes);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBK / 16; ++k)
            Wgmma<QBN>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) ? 1u : 0u);
          wgmma_commit();
          // this box's MMAs stay in flight; the previous box has been read once they are the only ones left
          wgmma_wait<1>();
          __syncwarp();
          if (kb > 0 && lane == 0) mbar_arrive(bar_empty + 8 * ((it - 1) % p.stages));
        }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * ((it - 1) % p.stages));
      auto key = [&](float a, float invn, float h, int col) {
        float s = a * invn;
        if constexpr (EUCLID) s = __fsub_rn(__fmul_rn(rq_s[col], s), h);
        return s;
      };
      // FILTER: row0 and row0 + 8 lie in one 32-row mask word; columns 4 j + 2 (lane % 4) + {0, 1} are one 8-byte load
      const uint32_t* mrow = nullptr;
      if constexpr (FILTER) mrow = p.mask + (size_t)(row0 >> 5) * p.mask_qs + 2 * (lane & 3);
      const int sh0 = (int)(row0 & 31), sh1 = sh0 + 8;
      if constexpr (STORE) {
#pragma unroll
        for (int a = 0; a < QBN / 2; ++a) {   // acc[a]: row row0 + 8 ((a >> 1) & 1), column 8 (a >> 2) + 2 (lane % 4) + (a & 1)
          const int h = (a >> 1) & 1;
          const int col = 8 * (a >> 2) + 2 * (lane & 3) + (a & 1);
          if ((h ? live1 : live0) && col < p.mask_qs)
            reinterpret_cast<float*>(p.cand)[(size_t)col * p.capg + row0 + 8 * h] = key(acc[a], h ? invn1 : invn0, 0.f, col);
        }
      } else if (p.thr_init == nullptr) {
        // Sampling pass.  The threshold only needs a LOWER bound of the k-th best score, and the k-th largest of ANY set
        // of distinct rows' scores is one: each warp contributes the best score among its 16 rows per query (two
        // registers, then a max over the 8 lanes that share a column), one 8-byte store per (warp, query) at slot
        // t * kSampleKeys + warp of the CTA's list.  FILTER: the best among its MATCHING rows; a warp without one
        // reports -inf, which can only lower the threshold.
        const int slot = t * kSampleKeys + warp;
#pragma unroll
        for (int j = 0; j < QBN / 4; j += 2) {   // acc[2 j .. 2 j + 3]: columns 4 j .. 4 j + 7
          uint2 mw = make_uint2(0u, 0u);
          if constexpr (FILTER) mw = __ldg(reinterpret_cast<const uint2*>(mrow + 4 * j));
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            bool m0 = live0, m1 = live1;
            if constexpr (FILTER) {
              const uint32_t w = e ? mw.y : mw.x;
              m0 = m0 && ((w >> sh0) & 1u);
              m1 = m1 && ((w >> sh1) & 1u);
            }
            const int col = 4 * j + 2 * (lane & 3) + e;
            const float s0 = m0 ? key(acc[2 * j + e], invn0, h0, col) : -INFINITY;
            const float s1 = m1 ? key(acc[2 * j + 2 + e], invn1, h1, col) : -INFINITY;
            uint32_t best = max(f32_orderable(s0), f32_orderable(s1));
            best = max(best, __shfl_xor_sync(0xffffffffu, best, 4));
            best = max(best, __shfl_xor_sync(0xffffffffu, best, 8));
            best = max(best, __shfl_xor_sync(0xffffffffu, best, 16));
            if (lane < 4) my_cand[(size_t)col * q_stride + slot] = ((unsigned long long)best << 32) | 0xffffffffull;
          }
        }
      } else {
        // Full pass.  About 0.3 % of the scores pass, so the test of every score is kept free of branches: one bit per
        // accumulator register, set when the row is live, score >= thr[col] (IEEE: -0 >= +0 holds, NaN fails) and,
        // FILTER, its match bit holds.  Bit a of the mask is acc[a]: row row0 + 8 ((a >> 1) & 1), column
        // 8 (a >> 2) + 2 (lane % 4) + (a & 1).  Only the set bits are then walked and appended, in the order of a.
        constexpr int kWords = (QBN / 2 + 31) / 32;
        uint32_t pass[kWords];
#pragma unroll
        for (int w = 0; w < kWords; ++w) pass[w] = 0u;
#pragma unroll
        for (int j = 0; j < QBN / 4; j += 2) {   // acc[2 j .. 2 j + 3]: columns 4 j .. 4 j + 7
          uint2 mw = make_uint2(0u, 0u);
          if constexpr (FILTER) mw = __ldg(reinterpret_cast<const uint2*>(mrow + 4 * j));
          // the thresholds of this thread's two columns: one 8-byte shared load serves all four scores of the step
          float2 tc;
          asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];"   // volatile: issued here, not hoisted into live registers
                       : "=f"(tc.x), "=f"(tc.y)
                       : "r"(thr_s + 4u * (4 * j + 2 * (lane & 3))));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int a = 2 * j + 2 * h + e;
              const int col = 4 * j + 2 * (lane & 3) + e;
              bool b = key(acc[a], h ? invn1 : invn0, h ? h1 : h0, col) >= (e ? tc.y : tc.x);
              if constexpr (FILTER) b = b && (((e ? mw.y : mw.x) >> (h ? sh1 : sh0)) & 1u);
              pass[a >> 5] |= (uint32_t)b << (a & 31);
            }
          }
        }
        // bits of row0 are a = 0, 1 mod 4, bits of row0 + 8 are a = 2, 3 mod 4
        const uint32_t live_bits = (live0 ? 0x33333333u : 0u) | (live1 ? 0xccccccccu : 0u);
#pragma unroll
        for (int w = 0; w < kWords; ++w) {
          uint32_t m = pass[w] & live_bits;
          while (m != 0u) {
            const int bit = __ffs(m) - 1;
            m &= m - 1u;
            const int a = 32 * w + bit;
            const int h = (a >> 1) & 1;
            const int col = 8 * (a >> 2) + 2 * (lane & 3) + (a & 1);
            const float score = key(acc_word_at(acc, w, bit), h ? invn1 : invn0, h ? h1 : h0, col);
            const int pos = atomicAdd(&cnt[col], 1);
            if (pos < p.capg) my_cand[(size_t)col * q_stride + pos] = make_key32(score, (uint32_t)(row0 + 8 * h));
          }
        }
      }
    }
  }
  if constexpr (STORE) return;
  __syncthreads();
  for (int i = threadIdx.x; i < QBN; i += blockDim.x) {
    const int c = p.thr_init == nullptr ? my_tiles * kSampleKeys : cnt[i];   // sampling pass: one key per warp and tile
    p.counts[(size_t)i * grid + cta] = min(c, p.capg);
    if (c > p.capg && p.fallback) p.fallback[i] = 1;   // nothing is dropped silently: brute force answers this query
  }
}

// ------------------------------------------------------------------------------------------------ select kernel
struct SelectParams {
  const unsigned long long* cand;   // [nq][grid][capg]
  const int32_t* counts;            // [nq][grid]
  int32_t grid, capg;
  int32_t nq;                       // real queries in this block (padded operand rows get a +inf threshold)
  int32_t mode;                     // 0 = write the safe threshold (sampling pass), 1 = window + exact stage + emit
  float* thr_out;                   // [rows] (mode 0)
  const float* eps;                 // [nq] error bound of the approximate scores (0 = all-zero query)
  int32_t* fallback;                // [nq] (mode 1)
  SlotView slot;                    // mode 1
  const float* q;                   // [nq][d_pad] the caller's fp32 queries
  int32_t k;
  int64_t* out_ids;
  double* out_scores;
  int32_t* out_counts;
  const int32_t* state;             // FILTER only: [nq] 1 = answered by the gather path (threshold +inf, no emit)
};

// One CTA per query.  A lower bound of the k-th best approximate key among the survivors of all CTAs by an MSB-first
// RADIX SELECT (8-bit digits, shared-memory histogram; the pass loop stops as soon as the bucket holding the k-th key
// is small -- the undecided low bits are taken as zero, which only widens the window).
//   mode 0 (sampling pass): threshold = that score - 2 eps.
//   mode 1: gather every survivor inside the window below it, exact fp64 re-score of all of them, emit k.
// Survivors are staged in shared memory when they fit (the normal case: ~0.3 % of the corpus); otherwise every pass
// streams them from HBM/L2 -- slower, still exact.  ST = SB_STORAGE_F32 / _U8: the exact stage scores the caller's rows.
template <bool FILTER, int ST>
__global__ void __launch_bounds__(kSelectThreads, 2) dense_select_kernel(const SelectParams p) {
  extern __shared__ __align__(16) uint8_t ssm[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(ssm);  // [kSelStage] staged survivors
  unsigned long long* top = keys + kSelStage;                             // [kSelTop]   window members
  unsigned long long* ek = top + kSelTop;                                 // [kSelTop]   exact keys      (mode 1)
  uint32_t* ei = reinterpret_cast<uint32_t*>(ek + kSelTop);               // [kSelTop]   rows            (mode 1)
  __shared__ double qq_s;
  __shared__ int s_prefix[kSelectThreads + 1];
  __shared__ int s_hist[256];
  __shared__ int s_scal[4];
  __shared__ int s_ntop;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5, qi = blockIdx.x;
  const int K = p.k, G = p.grid;
  if (p.mode == 0 && qi >= p.nq) {   // padded operand row: nothing may survive
    if (tid == 0) p.thr_out[qi] = INFINITY;
    return;
  }
  if constexpr (FILTER) {
    if (p.state[qi]) {   // answered by the gather path: nothing may survive, nothing to emit
      if (p.mode == 0 && tid == 0) p.thr_out[qi] = INFINITY;
      return;
    }
  }
  if (p.fallback[qi] != 0) {   // a list overflowed, or (mode 0) the query's keys are unbounded: brute force answers it
    if (p.mode == 0 && tid == 0) p.thr_out[qi] = INFINITY;
    return;
  }
  const int32_t* counts = p.counts + (size_t)qi * G;
  const unsigned long long* cand = p.cand + (size_t)qi * G * p.capg;
  // exclusive prefix of the per-CTA survivor counts (G <= blockDim): one element per thread
  {
    const int v = tid < G ? counts[tid] : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_hist[warp] = x;
    if (tid == 0) s_ntop = 0;
    __syncthreads();
    if (warp == 0) {
      int w = lane < nw ? s_hist[lane] : 0;
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      s_hist[32 + lane] = w;  // inclusive warp totals
    }
    __syncthreads();
    const int incl = x + (warp ? s_hist[32 + warp - 1] : 0);
    if (tid < G) s_prefix[tid] = incl - v;
    if (tid == G - 1) s_prefix[G] = incl;
    __syncthreads();
  }
  const int total = s_prefix[G];
  const bool staged = total <= kSelStage;
  if (staged) {
    for (int g = warp; g < G; g += nw) {
      const int c = s_prefix[g + 1] - s_prefix[g];
      const unsigned long long* src = cand + (size_t)g * p.capg;
      unsigned long long* dst = keys + s_prefix[g];
      for (int i = lane; i < c; i += 32) dst[i] = src[i];
    }
    __syncthreads();
  }
  // visit every survivor once: `body(key)`
#define SB_FOR_EACH_KEY(BODY)                                                       \
  if (staged) {                                                                     \
    for (int i_ = tid; i_ < total; i_ += nt) {                                      \
      const unsigned long long key = keys[i_];                                      \
      BODY                                                                          \
    }                                                                               \
  } else {                                                                          \
    for (int g_ = warp; g_ < G; g_ += nw) {                                         \
      const int c_ = s_prefix[g_ + 1] - s_prefix[g_];                               \
      const unsigned long long* src_ = cand + (size_t)g_ * p.capg;                  \
      for (int i_ = lane; i_ < c_; i_ += 32) {                                      \
        const unsigned long long key = src_[i_];                                    \
        BODY                                                                        \
      }                                                                             \
    }                                                                               \
  }

  unsigned long long prefix = 0ull, mask = 0ull;
  if (total > K) {
    int need = K;  // rank (from the top) of the key we are looking for inside the current bucket
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += nt) s_hist[i] = 0;
      __syncthreads();
      // warp-aggregated histogram update: in the leading passes nearly all keys share a digit, and per-key shared
      // atomics on one bin serialise; lanes with equal digits elect one lane to add their count
      SB_FOR_EACH_KEY(if ((key & mask) == prefix) {
        const int dgt = (int)((key >> shift) & 0xffull);
        const unsigned grp = __match_any_sync(__activemask(), dgt);
        if ((int)(threadIdx.x & 31) == __ffs(grp) - 1) atomicAdd(&s_hist[dgt], __popc(grp));
      })
      __syncthreads();
      if (warp == 0) warp_select_bin<true>(s_hist, need, lane, s_scal);
      __syncthreads();
      prefix |= (unsigned long long)s_scal[0] << shift;
      mask |= 0xffull << shift;
      need = s_scal[1];
      const int bucket = s_scal[2];
      __syncthreads();
      if (bucket <= 16) break;
    }
  }
  // `prefix` (undecided low bits zero) <= the k-th best key; total <= k: every survivor is a member (prefix = 0)
  const float eps = p.eps[qi];
  const unsigned long long lo_key = total > K ? window_lo_key(prefix, eps) : 0ull;
  if (p.mode == 0) {
    // fewer than k sampled rows: no threshold.  The score field of lo_key is (k-th best of the sample) - 2 eps.
    if (tid == 0) p.thr_out[qi] = total > K ? key32_score(lo_key) : -INFINITY;
    return;
  }
  SB_FOR_EACH_KEY(if (key >= lo_key) {
    const int at = atomicAdd(&s_ntop, 1);
    if (at < kSelTop) top[at] = key;
  })
#undef SB_FOR_EACH_KEY
  __syncthreads();
  const int ntop = s_ntop;
  if (ntop > kSelTop) {
    if (tid == 0) p.fallback[qi] = 1;
    return;
  }
  int P = 32;
  while (P < ntop) P <<= 1;
  const RescoreArgs ra{p.slot, p.q + (size_t)qi * p.slot.d_pad, p.k, p.out_ids + (size_t)qi * p.k,
                       p.out_scores + (size_t)qi * p.k, p.out_counts + qi};
  // the staged survivors are dead (the window lives in `top`): their shared memory becomes the query staging area
  rescore_and_emit<ST>(top, ntop, P, ek, ei, &qq_s, reinterpret_cast<float*>(keys), ra);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// fp16 K-major operand (SWIZZLE_128B, 64-column boxes), or with u8 the uint8 corpus (64-byte boxes, no swizzle)
int encode_map(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols, int box_rows, bool u8 = false) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* pfn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &pfn, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(pfn);
  }
  SB_REQUIRE(fn != nullptr, SB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * (u8 ? 1 : 2)};
  cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, u8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr),
                  dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  u8 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SB_REQUIRE(r == CUDA_SUCCESS, SB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return SB_OK;
}

// the slot's cached corpus map (ix.tm_rows), (re)built when rows or n_pad change
int corpus_map(DenseIndex& ix) {
  const bool u8 = ix.storage == SB_STORAGE_U8;
  const void* corpus = u8 ? (const void*)ix.rows8 : (const void*)ix.rows;
  if (ix.tm_rows_ptr != corpus || ix.tm_n_pad != ix.n_pad) {
    int rc;
    if ((rc = encode_map(reinterpret_cast<CUtensorMap*>(ix.tm_rows), corpus, ix.n_pad, ix.d_pad, kTileRows, u8)))
      return rc;
    ix.tm_rows_ptr = corpus;
    ix.tm_n_pad = ix.n_pad;
  }
  return SB_OK;
}

// ring stages of a QBN-query group: corpus box + query box each, capped by SB_DENSE_STAGES.  Per query: threshold and
// count, and for Euclid the query norm r.  A uint8 corpus box is half the size (at QBN = 256: 40 KB stages, five fit).
size_t mma_per_query(bool euclid) { return euclid ? 12 : 8; }
int mma_stages(const sb_ctx* ctx, int qbn, bool euclid = false, bool u8 = false) {
  const size_t stage = (u8 ? kATileBytesU8 : kATileBytes) + (size_t)qbn * kBK * 2 + 16;   // + its full / empty barriers
  const size_t fixed = 1024 + (size_t)qbn * mma_per_query(euclid); // alignment slack + per-query values
  return std::min((int)((ctx->smem_optin - fixed) / stage), ctx->dense_max_stages);
}
size_t mma_smem(int qbn, int stages, bool euclid, bool u8 = false) {
  return 1024 + (size_t)stages * ((u8 ? kATileBytesU8 : kATileBytes) + (size_t)qbn * kBK * 2 + 16) +
         (size_t)qbn * mma_per_query(euclid);
}

template <int QBN, bool FILTER, bool EUCLID, int ST, bool STORE = false>
int launch_mma(const CUtensorMap& tm_rows, const CUtensorMap& tm_q, const MmaScanParams& mp, int grid, size_t smem,
               cudaStream_t st) {
  auto kern = dense_scan_mma_kernel<QBN, FILTER, EUCLID, ST, STORE>;
  SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, kMmaThreads, smem, st>>>(tm_rows, tm_q, mp);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

// ST: SB_STORAGE_U8 for a uint8 corpus; float16 and float32 slots scan the same fp16 rows (SB_STORAGE_F16)
template <bool FILTER, bool EUCLID, int ST, bool STORE = false>
int dispatch_mma(int qbn, const CUtensorMap& tm_rows, const CUtensorMap& tm_q, const MmaScanParams& mp, int grid,
                 size_t smem, cudaStream_t st) {
  switch (qbn) {
    case 16: return launch_mma<16, FILTER, EUCLID, ST, STORE>(tm_rows, tm_q, mp, grid, smem, st);
    case 32: return launch_mma<32, FILTER, EUCLID, ST, STORE>(tm_rows, tm_q, mp, grid, smem, st);
    case 64: return launch_mma<64, FILTER, EUCLID, ST, STORE>(tm_rows, tm_q, mp, grid, smem, st);
    case 128: return launch_mma<128, FILTER, EUCLID, ST, STORE>(tm_rows, tm_q, mp, grid, smem, st);
    case 256: return launch_mma<256, FILTER, EUCLID, ST, STORE>(tm_rows, tm_q, mp, grid, smem, st);
  }
  sb_set_error("dense_mma: unsupported query block %d", qbn);
  return SB_ERR_UNSUPPORTED;
}


// ------------------------------------------------------------------------------------------------ recommendation (K1j)
// The scan in STORE mode leaves key a_j(x) of every (example j, row x) of a pass.  With |a_j(x) - s_j(x) / c_j| <= eps_j
// (c_j = ||e_j|| for Dot, 1 for Cosine), s_j(x) lies in [c_j a_j - delta_j, c_j a_j + delta_j], delta_j = c_j eps_j.  The
// merged score is non-decreasing in every positive and non-increasing in every negative similarity (best_score across
// its jump at p = n too), so its interval is the merge at the two corners, widened by the fp64 rounding.  The exact top-k lies in W = {x : hi(x) >= the k-th largest lo}; every member is re-scored in fp64.
constexpr int kRecoThreads = 1024;
constexpr int kRecoFbBest = 1024;                  // >= k
constexpr int64_t kRecoKeyBudget = 1ll << 30;      // bytes of keys of one pass (examples x n_pad fp32)
constexpr int64_t kRecoBoundBudget = 1ll << 29;    // bytes of intervals of one pass (requests x n_pad x 16)

__device__ __forceinline__ double reco_g(double x) { return 0.5 * (x / (1.0 + fabs(x)) + 1.0); }
// best_score of (p, n); ties p == n take the negative branch
__device__ __forceinline__ double reco_best(double p, double n) { return p > n ? reco_g(p) : -reco_g(n); }

// ||e_j|| in fp64 as query_norm_cta computes it, and (c_j, delta_j); one warp per example
__global__ void __launch_bounds__(256) dense_reco_norms_kernel(const float* ex, int M, int d_pad, int metric,
                                                               const float* eps, double* qn, double* cd) {
  const int j = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (j >= M) return;
  double s = 0.0;
  for (int i = lane; i < d_pad; i += 32) {
    const double v = (double)ex[(size_t)j * d_pad + i];
    s += v * v;
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const double nrm = sqrt(s);
    const double c = metric == SB_METRIC_DOT ? nrm : 1.0;
    qn[j] = nrm;
    cd[2 * j] = c;
    cd[2 * j + 1] = c * (double)eps[j];
  }
}

struct RecoCombineParams {
  const float* keys;      // [examples of the pass][ld]
  int64_t ld, n;
  int32_t e0, r0;         // first example / request of the pass
  const RecoReq* req;
  const double* cd;       // [M][2] c_j, delta_j
  const uint32_t* mask;   // filtered passes: bit (row % 32) of mask[(row / 32) * mask_qs + request - r0]
  int32_t mask_qs;
  unsigned long long* lo; // [requests of the pass][ld] orderable fp64 lower bound; 0 = the row does not match
  double* hi;             // [requests of the pass][ld] upper bound
};

__global__ void __launch_bounds__(256) dense_reco_combine_kernel(const RecoCombineParams p) {
  const int rl = blockIdx.y;
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= p.n) return;
  const RecoReq q = p.req[p.r0 + rl];
  bool match = true;
  if (p.mask) match = (p.mask[(size_t)(row >> 5) * p.mask_qs + rl] >> (row & 31)) & 1u;
  unsigned long long lo_key = 0ull;
  double hi_d = -INFINITY;
  if (match) {
    double plo = -INFINITY, phi = -INFINITY, nlo = -INFINITY, nhi = -INFINITY, slo = 0.0, shi = 0.0, scale = 0.0;
    const float* kc = p.keys + (size_t)(q.ex0 - p.e0) * p.ld + row;
    for (int j = 0; j < q.m; ++j) {
      const double c = p.cd[2 * (q.ex0 + j)], d = p.cd[2 * (q.ex0 + j) + 1];
      const double s = c * (double)__ldg(kc + (size_t)j * p.ld);
      const double w = 1e-12 * (fabs(s) + d);   // covers the fp64 rounding of s and s -+ d
      const double a = s - d - w, b = s + d + w;
      if (j < q.n_pos) {
        plo = fmax(plo, a);
        phi = fmax(phi, b);
        slo += a;
        shi += b;
      } else {
        nlo = fmax(nlo, a);
        nhi = fmax(nhi, b);
        slo -= b;
        shi -= a;
      }
      scale += fabs(s) + d;
    }
    // fp64 rounding: of g, inside 1e-15 (g <= 1); of a sum of <= 256 terms, inside 1e-12 (1 + scale).  The intervals
    // stay fp64: a Dot best_score saturates g near 1, where fp32 would merge every row into a few values.
    const bool best = q.strategy == SB_RECO_BEST_SCORE;
    const double slack = best ? 1e-15 : 1e-12 * (1.0 + scale);
    const double lo = (best ? reco_best(plo, nhi) : slo) - slack;
    hi_d = (best ? reco_best(phi, nlo) : shi) + slack;
    lo_key = f64_orderable(lo);
  }
  p.lo[(size_t)rl * p.ld + row] = lo_key;
  p.hi[(size_t)rl * p.ld + row] = hi_d;
}

struct RecoSelectParams {
  const unsigned long long* lo;
  const double* hi;
  int64_t ld, n;
  int32_t r0;
  const RecoReq* req;
  const float* ex;              // [M][d_pad] the caller's fp32 examples
  const double* qn;             // [M] ||e_j||
  const int32_t* ex_fb;         // [M] raised by the query preparation: the keys of e_j are not bounded
  SlotView slot;
  int32_t k;
  int32_t* fallback;            // [R]
  int64_t* out_ids;             // [R][k]
  double* out_scores;
  int32_t* out_counts;          // [R]
  const uint32_t* mask;         // fallback: as RecoCombineParams
  int32_t mask_qs;
  unsigned long long* counter;  // fallback: requests answered by brute force
};

// exact merged score of one row (one full warp; every lane returns it)
template <int ST>
__device__ __forceinline__ double reco_exact_row(const RecoSelectParams& p, const RecoReq& q, uint32_t row, int lane) {
  double sp = 0.0, sn = 0.0, pm = -INFINITY, nm = -INFINITY;
  for (int j = 0; j < q.m; ++j) {
    const int e = q.ex0 + j;
    const double s = exact_key_row<ST>(p.slot, row, p.ex + (size_t)e * p.slot.d_pad, p.qn[e], lane);
    if (j < q.n_pos) {
      sp += s;
      pm = fmax(pm, s);
    } else {
      sn += s;
      nm = fmax(nm, s);
    }
  }
  return q.strategy == SB_RECO_BEST_SCORE ? reco_best(pm, nm) : sp - sn;
}

// One CTA per request of the pass: the k-th largest lower bound by an MSB-first radix select over the request's rows,
// the window {hi >= it}, the exact re-score of the window and the emit.  A window over kSelTop raises the fallback flag.
template <int ST>
__global__ void __launch_bounds__(kRecoThreads, 1) dense_reco_select_kernel(const RecoSelectParams p) {
  __shared__ uint32_t top[kSelTop];
  __shared__ unsigned long long ek[kSelTop];
  __shared__ uint32_t ei[kSelTop];
  __shared__ int s_hist[256];
  __shared__ int s_scal[4];
  __shared__ int s_cnt;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x, nw = nt >> 5;
  const int rl = blockIdx.x, r = p.r0 + rl;
  const RecoReq q = p.req[r];
  if (tid == 0) {
    int f = 0;
    for (int j = 0; j < q.m; ++j) f |= p.ex_fb[q.ex0 + j];
    s_cnt = f;
  }
  __syncthreads();
  if (s_cnt != 0) {
    if (tid == 0) p.fallback[r] = 1;
    return;
  }
  __syncthreads();
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  const unsigned long long* lo = p.lo + (size_t)rl * p.ld;
  const double* hi = p.hi + (size_t)rl * p.ld;
  {
    int c = 0;
    for (int64_t i = tid; i < p.n; i += nt) c += lo[i] != 0ull;
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0 && c) atomicAdd(&s_cnt, c);
  }
  __syncthreads();
  const int total = s_cnt;
  double thr = -INFINITY;   // at most k candidates: every one is a member
  if (total > p.k) {
    unsigned long long prefix = 0ull, msk = 0ull;
    int need = p.k;
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += nt) s_hist[i] = 0;
      __syncthreads();
      for (int64_t i = tid; i < p.n; i += nt) {
        const unsigned long long key = lo[i];
        if (key != 0ull && (key & msk) == prefix) {
          const int dgt = (int)((key >> shift) & 0xffull);
          const unsigned grp = __match_any_sync(__activemask(), dgt);
          if (lane == __ffs(grp) - 1) atomicAdd(&s_hist[dgt], __popc(grp));
        }
      }
      __syncthreads();
      if (warp == 0) warp_select_bin<true>(s_hist, need, lane, s_scal);
      __syncthreads();
      prefix |= (unsigned long long)s_scal[0] << shift;
      msk |= 0xffull << shift;
      need = s_scal[1];
      __syncthreads();
    }
    thr = orderable_f64(prefix);   // the k-th largest lower bound
  }
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  for (int64_t i = tid; i < p.n; i += nt)
    if (lo[i] != 0ull && hi[i] >= thr) {
      const int at = atomicAdd(&s_cnt, 1);
      if (at < kSelTop) top[at] = (uint32_t)i;
    }
  __syncthreads();
  const int ntop = s_cnt;
  if (ntop > kSelTop) {
    if (tid == 0) p.fallback[r] = 1;
    return;
  }
  int P = 32;
  while (P < ntop) P <<= 1;
  for (int c = warp; c < P; c += nw) {
    unsigned long long okey = 0ull;
    uint32_t row = 0xffffffffu;
    if (c < ntop) {
      row = top[c];
      okey = f64_orderable(reco_exact_row<ST>(p, q, row, lane));
      if (okey == 0ull) okey = 1ull;   // 0 is reserved for "empty"
    }
    if (lane == 0) {
      ek[c] = okey;
      ei[c] = row;
    }
  }
  __syncthreads();
  sort_exact_pairs(ek, ei, P, tid, nt);
  const RescoreArgs ra{p.slot, nullptr, p.k, p.out_ids + (size_t)r * p.k, p.out_scores + (size_t)r * p.k,
                       p.out_counts + r};
  emit_exact_pairs(ek, ei, P, ra);
}

// One CTA per FLAGGED request of the pass: the merged score of every matching row in fp64, 1024 rows per round folded
// into the running best list (as dense_exact_fallback_kernel).
template <int ST>
__global__ void __launch_bounds__(kRecoThreads, 1) dense_reco_fallback_kernel(const RecoSelectParams p) {
  const int rl = blockIdx.x, r = p.r0 + rl;
  if (p.fallback[r] == 0) return;
  __shared__ unsigned long long ek[2 * kRecoFbBest];
  __shared__ uint32_t ei[2 * kRecoFbBest];
  __shared__ int s_beats;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x, nw = nt >> 5;
  if (tid == 0) atomicAdd(p.counter, 1ull);
  const RecoReq q = p.req[r];
  for (int i = tid; i < 2 * kRecoFbBest; i += nt) {
    ek[i] = 0ull;
    ei[i] = 0xffffffffu;
  }
  __syncthreads();
  for (int64_t r0 = 0; r0 < p.n; r0 += kRecoFbBest) {
    if (tid == 0) s_beats = 0;
    __syncthreads();
    const unsigned long long kth = ek[p.k - 1];
    bool beat = false;
    for (int c = warp; c < kRecoFbBest; c += nw) {
      const int64_t row = r0 + c;
      bool match = row < p.n;
      if (match && p.mask) match = (p.mask[(size_t)(row >> 5) * p.mask_qs + rl] >> (row & 31)) & 1u;
      unsigned long long okey = 0ull;
      if (match) {
        okey = f64_orderable(reco_exact_row<ST>(p, q, (uint32_t)row, lane));
        if (okey == 0ull) okey = 1ull;
      }
      if (lane == 0) {
        ek[kRecoFbBest + c] = okey;
        ei[kRecoFbBest + c] = row < p.n ? (uint32_t)row : 0xffffffffu;
        beat |= okey > kth;
      }
    }
    if (beat) s_beats = 1;
    __syncthreads();
    if (s_beats) sort_exact_pairs(ek, ei, 2 * kRecoFbBest, tid, nt);
    __syncthreads();
  }
  const RescoreArgs ra{p.slot, nullptr, p.k, p.out_ids + (size_t)r * p.k, p.out_scores + (size_t)r * p.k,
                       p.out_counts + r};
  emit_exact_pairs(ek, ei, kRecoFbBest, ra);
}

}  // namespace

bool dense_mma_eligible(const sb_ctx* ctx, const DenseIndex& ix, int B) {
  if (B < 16) return false;
  if (ix.d_pad % kBK != 0 || ix.n_pad % kTileRows != 0) return false;
  if (ix.n < 64 * kTileRows) return false;  // tiny corpora: the CUDA-core scan is already launch bound
  return mma_stages(ctx, kQbnMax) >= 3;     // shared memory does not depend on d
}

int dense_mma_topk_enqueue(sb_ctx* ctx, DenseIndex& ix, const float* q_pad, int B, int k, int64_t* out_ids,
                           double* out_scores, int32_t* out_counts, cudaStream_t st, const DenseFilter* flt) {
  const int kb_count = ix.d_pad / kBK;
  const int total_tiles = (int)(ix.n_pad / kTileRows);
  const int gsz = kQbnMax;                          // operand rows per group
  const int grid = std::min(ctx->num_sms, total_tiles);
  // filtered: a fraction phi of the rows matches the group's sparsest scanned query; a 16-row warp holds a matching row
  // with probability hit = 1 - (1 - phi)^16, and then ~ m_eff = 16 phi / hit of them
  const double phi = flt ? std::min(1.0, (double)std::max<int64_t>(flt->c_min, 1) / (double)ix.n) : 1.0;
  const double hit = flt ? 1.0 - pow(1.0 - phi, (double)kSampleRows) : 1.0;
  const double m_eff = flt ? (double)kSampleRows * phi / hit : (double)kSampleRows;
  // sampling pass geometry: a few tiles per CTA spread evenly over the corpus; every warp of a sampled tile reports the
  // best of its 16 rows, so a query gets n_s = kSampleKeys * sample_tiles keys -- aim for n_s >= 4 k (filtered: 4 k
  // keys that come from a matching row, up to a sampling pass over the whole corpus)
  const int per_cta = flt ? std::max(ctx->dense_sample_per_cta,
                                     (int)ceil(4.0 * k / ((double)kSampleKeys * hit * grid)))
                          : std::max(ctx->dense_sample_per_cta, std::min(8, (4 * k / kSampleKeys + grid - 1) / grid));
  const int sample_tiles = (int)std::min<int64_t>((int64_t)per_cta * grid, total_tiles);
  const int sample_step = total_tiles / sample_tiles;
  const int sgrid = std::min(grid, sample_tiles);
  // per-(CTA, query) list capacity.  Sampling pass: kSampleKeys keys per sampled tile of the CTA.  Full pass: the
  // threshold is the k-th best of n_s maxima of 16 rows, passed by a fraction p of the rows with (1 - p)^16 = 1 - k / n_s;
  // 8x the expected rows_per_cta * p plus slack.  An overflowing list raises the query's fallback flag, so the capacity
  // only trades memory against the odds of a brute-force answer; no threshold at all (k >= n_s) means every row survives.
  // Filtered: n_s * hit real keys over groups of m_eff matching rows, passed by a fraction p of the phi * rows_per_cta
  // matching rows; for every scanned query (phi >= the smallest) the expected survivors are at most this many.
  const int64_t worst = (int64_t)((total_tiles + grid - 1) / grid + 1) * kTileRows;
  const int64_t samp_keys = (int64_t)((sample_tiles + sgrid - 1) / sgrid + 1) * kSampleKeys;
  const double f = (double)k / ((double)kSampleKeys * sample_tiles * hit);
  const double pass = f >= 0.95 ? 1.0 : -log(1.0 - f) / m_eff;
  const int64_t expect = (int64_t)((double)worst * phi * pass) + 1;
  const int capg = (int)std::min<int64_t>(worst, std::max<int64_t>(8 * expect + 256, samp_keys));
  int rc;
  SB_REQUIRE(grid <= kSelectThreads, SB_ERR_UNSUPPORTED, "dense_mma: %d CTAs exceed the select kernel's prefix width", grid);
  const int n_groups = (B + gsz - 1) / gsz;
  const size_t cand_per_group = (size_t)gsz * grid * capg * 8;
  int gmax = (int)std::max<size_t>(1, (size_t)(1024ull << 20) / cand_per_group);
  gmax = std::min(gmax, n_groups);
  // scratch: fp16 operand rows | thresholds + counts | survivors
  if ((rc = ctx->misc2_dev.reserve((size_t)n_groups * gsz * ix.d_pad * 2 + 256))) return rc;
  if ((rc = ctx->misc3_dev.reserve(((size_t)gsz * 4 + (size_t)gsz * grid * 4) * gmax + 256))) return rc;
  if ((rc = ctx->cand_dev.reserve(cand_per_group * gmax))) return rc;
  __half* q16 = ctx->misc2_dev.as<__half>();
  float* thr = ctx->misc3_dev.as<float>();
  int32_t* counts = reinterpret_cast<int32_t*>(thr + (size_t)gsz * gmax);
  unsigned long long* cand = ctx->cand_dev.as<unsigned long long>();
  const bool u8 = ix.storage == SB_STORAGE_U8;
  if ((rc = corpus_map(ix))) return rc;
  const CUtensorMap& tm_rows = *reinterpret_cast<const CUtensorMap*>(ix.tm_rows);
  const size_t sel_smem = (size_t)kSelStage * 8 + (size_t)kSelTop * 20 + 64;
  auto sel_kern = flt ? dense_select_kernel<true, SB_STORAGE_F16> : dense_select_kernel<false, SB_STORAGE_F16>;
  if (ix.storage == SB_STORAGE_F32)
    sel_kern = flt ? dense_select_kernel<true, SB_STORAGE_F32> : dense_select_kernel<false, SB_STORAGE_F32>;
  else if (u8)
    sel_kern = flt ? dense_select_kernel<true, SB_STORAGE_U8> : dense_select_kernel<false, SB_STORAGE_U8>;
  SB_CUDA(cudaFuncSetAttribute(sel_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_smem));
  auto launch_select = [&](int nblocks, const SelectParams& s) {
    sel_kern<<<nblocks, kSelectThreads, sel_smem, st>>>(s);
  };
  const bool euclid = ix.metric == SB_METRIC_EUCLID;   // Cosine and Dot run the same (acc * scale) kernels
  auto run_mma = [&](int qbn, const CUtensorMap& tm_q, const MmaScanParams& m, int g, size_t smem) {
    constexpr int F16 = SB_STORAGE_F16, U8 = SB_STORAGE_U8;
    if (u8) {
      if (euclid)
        return flt ? dispatch_mma<true, true, U8>(qbn, tm_rows, tm_q, m, g, smem, st)
                   : dispatch_mma<false, true, U8>(qbn, tm_rows, tm_q, m, g, smem, st);
      return flt ? dispatch_mma<true, false, U8>(qbn, tm_rows, tm_q, m, g, smem, st)
                 : dispatch_mma<false, false, U8>(qbn, tm_rows, tm_q, m, g, smem, st);
    }
    if (euclid)
      return flt ? dispatch_mma<true, true, F16>(qbn, tm_rows, tm_q, m, g, smem, st)
                 : dispatch_mma<false, true, F16>(qbn, tm_rows, tm_q, m, g, smem, st);
    return flt ? dispatch_mma<true, false, F16>(qbn, tm_rows, tm_q, m, g, smem, st)
               : dispatch_mma<false, false, F16>(qbn, tm_rows, tm_q, m, g, smem, st);
  };
  // normalised fp16 operand rows of the whole batch (rows beyond B are zero), eps, cleared fallback flags (and r)
  float *eps = nullptr, *rq = nullptr;
  int32_t* fb = nullptr;
  if ((rc = dense_prep_queries(ctx, ix, q_pad, B, n_groups * gsz, /*mma=*/true, nullptr, q16, &eps, &fb, &rq, st)))
    return rc;

  for (int c0 = 0; c0 < B; c0 += gmax * gsz) {
    const int nq_chunk = std::min(B - c0, gmax * gsz);   // real queries of this chunk of groups
    const int ng = (nq_chunk + gsz - 1) / gsz;
    struct Group { int qbn, nq; CUtensorMap tm_q; size_t smem; int stages; };
    std::vector<Group> gs((size_t)ng);
    int rows_total = 0;  // operand rows of the chunk (padding only at the very end)
    for (int g = 0; g < ng; ++g) {
      Group& G = gs[(size_t)g];
      const int left = nq_chunk - g * gsz;
      __half* q16g = q16 + (size_t)(c0 + g * gsz) * ix.d_pad;
      G.qbn = gsz;
      while (G.qbn > 16 && G.qbn / 2 >= left) G.qbn >>= 1;
      G.nq = std::min(G.qbn, left);
      if ((rc = encode_map(&G.tm_q, q16g, G.qbn, ix.d_pad, G.qbn))) return rc;
      G.stages = mma_stages(ctx, G.qbn, euclid, u8);
      G.smem = mma_smem(G.qbn, G.stages, euclid, u8);
      rows_total = g * gsz + G.qbn;
    }
    MmaScanParams mp;
    mp.inv_norm = ix.inv_norm;
    mp.n = ix.n;
    mp.kb_count = kb_count;
    mp.capg = capg;
    mp.prefetch = ctx->dense_prefetch;
    mp.mask_qs = flt ? flt->qs : 0;
    mp.hh = ix.hh;
    SelectParams sp;
    sp.cand = cand;
    sp.counts = counts;
    sp.capg = capg;
    sp.nq = nq_chunk;
    sp.thr_out = thr;
    sp.eps = eps + c0;
    sp.fallback = fb + c0;
    sp.slot = slot_view(ix);
    sp.q = q_pad + (size_t)c0 * ix.d_pad;
    sp.k = k;
    sp.out_ids = out_ids + (size_t)c0 * k;
    sp.out_scores = out_scores + (size_t)c0 * k;
    sp.out_counts = out_counts + c0;
    sp.state = flt ? flt->state + c0 : nullptr;
    // (1) sampling passes -> safe thresholds for every query of the chunk (one select launch).  The kernel writes list
    // slot `cta` of [row][launch grid][capg], so every group is launched with exactly sgrid CTAs.
    mp.thr_init = nullptr;
    mp.fallback = nullptr;   // capg >= the sampled rows of a CTA: the sampling pass cannot overflow
    mp.num_tiles = sample_tiles;
    mp.tile_first = 0;
    mp.tile_step = sample_step;
    {
      ProfScope ps(ctx, SB_PROF_DENSE_SAMPLE, st, ng + 1);   // the sampling passes + their threshold select, as one span
      for (int g = 0; g < ng; ++g) {
        const Group& G = gs[(size_t)g];
        mp.cand = cand + (size_t)g * gsz * sgrid * capg;
        mp.counts = counts + (size_t)g * gsz * sgrid;
        mp.stages = G.stages;
        mp.mask = flt ? flt->mask + c0 + (size_t)g * gsz : nullptr;
        mp.rq = rq ? rq + c0 + (size_t)g * gsz : nullptr;
        if ((rc = run_mma(G.qbn, G.tm_q, mp, sgrid, G.smem))) return rc;
      }
      sp.grid = sgrid;
      sp.mode = 0;
      launch_select(rows_total, sp);
    }
    SB_CUDA(cudaGetLastError());
    // (2) the full passes, then one select + exact re-score launch for the chunk
    mp.num_tiles = total_tiles;
    mp.tile_first = 0;
    mp.tile_step = 1;
    for (int g = 0; g < ng; ++g) {
      const Group& G = gs[(size_t)g];
      mp.thr_init = thr + (size_t)g * gsz;
      mp.fallback = fb + c0 + (size_t)g * gsz;
      mp.cand = cand + (size_t)g * gsz * grid * capg;
      mp.counts = counts + (size_t)g * gsz * grid;
      mp.stages = G.stages;
      mp.mask = flt ? flt->mask + c0 + (size_t)g * gsz : nullptr;
      mp.rq = rq ? rq + c0 + (size_t)g * gsz : nullptr;
      ProfScope ps(ctx, SB_PROF_DENSE_SCAN, st);
      if ((rc = run_mma(G.qbn, G.tm_q, mp, grid, G.smem))) return rc;
    }
    sp.grid = grid;
    sp.mode = 1;
    {
      ProfScope ps(ctx, SB_PROF_DENSE_MERGE, st);
      launch_select(nq_chunk, sp);
    }
    SB_CUDA(cudaGetLastError());
  }
  return dense_fallback_enqueue(ctx, ix, q_pad, B, k, fb, out_ids, out_scores, out_counts, st, flt);
}

// Recommendation (DESIGN.md K1j): requests packed into passes of <= 256 examples (fewer on slots whose keys would pass
// kRecoKeyBudget, never fewer than the largest request), one STORE-mode scan per pass, then per pass the intervals, the
// select + exact stage and the brute force of the flagged requests.
int dense_reco_enqueue(sb_ctx* ctx, DenseIndex& ix, const float* ex_pad, int M, const RecoReq* req, int R, int k,
                       const int32_t* p_off, const sb_pred* prog, const int32_t* pool, int64_t* out_ids,
                       double* out_scores, int32_t* out_counts, cudaStream_t st) {
  const bool u8 = ix.storage == SB_STORAGE_U8;
  const int64_t n_pad = ix.n_pad;
  auto align_up = [](size_t v, size_t a) { return (v + a - 1) / a * a; };
  int m_max = 1;
  for (int r = 0; r < R; ++r) m_max = std::max(m_max, req[r].m);
  const int e_cap = std::max(m_max, (int)std::min<int64_t>(kQbnMax, std::max<int64_t>(16, kRecoKeyBudget / (4 * n_pad))));
  const int r_cap = (int)std::min<int64_t>(kQbnMax, std::max<int64_t>(1, kRecoBoundBudget / (16 * n_pad)));
  // scratch: fp16 operand rows | qn [M] | (c, delta) [M] | requests [R] | fallback [R] | keys | lo | hi
  const size_t o_qn = align_up((size_t)(M + kQbnMax) * ix.d_pad * 2, 256);
  const size_t o_cd = o_qn + align_up((size_t)M * 8, 256);
  const size_t o_req = o_cd + align_up((size_t)M * 16, 256);
  const size_t o_fb = o_req + align_up((size_t)R * sizeof(RecoReq), 256);
  const size_t o_keys = o_fb + align_up((size_t)R * 4, 256);
  const size_t o_lo = o_keys + align_up((size_t)e_cap * n_pad * 4, 256);
  const size_t o_hi = o_lo + (size_t)r_cap * n_pad * 8;
  int rc;
  if ((rc = ctx->reco_dev.reserve(o_hi + (size_t)r_cap * n_pad * 8))) return rc;
  uint8_t* base = ctx->reco_dev.as<uint8_t>();
  __half* q16 = reinterpret_cast<__half*>(base);
  double* qn = reinterpret_cast<double*>(base + o_qn);
  double* cd = reinterpret_cast<double*>(base + o_cd);
  RecoReq* req_d = reinterpret_cast<RecoReq*>(base + o_req);
  int32_t* fb = reinterpret_cast<int32_t*>(base + o_fb);
  float* keys = reinterpret_cast<float*>(base + o_keys);
  unsigned long long* lo = reinterpret_cast<unsigned long long*>(base + o_lo);
  double* hi = reinterpret_cast<double*>(base + o_hi);
  SB_CUDA(cudaMemcpyAsync(req_d, req, (size_t)R * sizeof(RecoReq), cudaMemcpyHostToDevice, st));
  SB_CUDA(cudaMemsetAsync(fb, 0, (size_t)R * 4, st));
  if (ctx->fb_count_dev.cap == 0) {
    if ((rc = ctx->fb_count_dev.reserve(8))) return rc;
    SB_CUDA(cudaMemsetAsync(ctx->fb_count_dev.p, 0, 8, st));
  }
  float *eps = nullptr, *rq = nullptr;
  int32_t* ex_fb = nullptr;
  if ((rc = dense_prep_queries(ctx, ix, ex_pad, M, M + kQbnMax, /*mma=*/true, nullptr, q16, &eps, &ex_fb, &rq, st)))
    return rc;
  dense_reco_norms_kernel<<<(M + 7) / 8, 256, 0, st>>>(ex_pad, M, ix.d_pad, ix.metric, eps, qn, cd);
  SB_CUDA(cudaGetLastError());
  ctx->launches += 1;
  if ((rc = corpus_map(ix))) return rc;
  const CUtensorMap& tm_rows = *reinterpret_cast<const CUtensorMap*>(ix.tm_rows);
  const int total_tiles = (int)(n_pad / kTileRows);
  const int grid = std::min(ctx->num_sms, total_tiles);
  auto sel_kern = u8 ? dense_reco_select_kernel<SB_STORAGE_U8>
                  : ix.storage == SB_STORAGE_F32 ? dense_reco_select_kernel<SB_STORAGE_F32>
                                                 : dense_reco_select_kernel<SB_STORAGE_F16>;
  auto fb_kern = u8 ? dense_reco_fallback_kernel<SB_STORAGE_U8>
                 : ix.storage == SB_STORAGE_F32 ? dense_reco_fallback_kernel<SB_STORAGE_F32>
                                                : dense_reco_fallback_kernel<SB_STORAGE_F16>;
  for (int r0 = 0; r0 < R;) {
    int r1 = r0 + 1, me = req[r0].m;
    while (r1 < R && r1 - r0 < r_cap && me + req[r1].m <= e_cap) me += req[r1++].m;
    const int nr = r1 - r0, e0 = req[r0].ex0;
    const uint32_t* mask = nullptr;
    int qs = 0;
    if (p_off && p_off[r1] > p_off[r0] &&
        (rc = dense_where_mask(ctx, ix, p_off, prog, pool, r0, nr, &mask, &qs, st)))
      return rc;
    int qbn = 16;
    while (qbn < me) qbn <<= 1;
    CUtensorMap tm_q;
    if ((rc = encode_map(&tm_q, q16 + (size_t)e0 * ix.d_pad, qbn, ix.d_pad, qbn))) return rc;
    MmaScanParams mp = {};
    mp.inv_norm = ix.inv_norm;
    mp.n = ix.n;
    mp.kb_count = (ix.d_pad + kBK - 1) / kBK;   // a partial last box is zero-filled by the TMA unit
    mp.num_tiles = total_tiles;
    mp.tile_first = 0;
    mp.tile_step = 1;
    mp.stages = mma_stages(ctx, qbn, false, u8);
    mp.prefetch = ctx->dense_prefetch;
    mp.cand = reinterpret_cast<unsigned long long*>(keys);   // STORE: the key buffer, row stride capg
    mp.capg = (int32_t)n_pad;
    mp.mask_qs = me;
    const size_t smem = mma_smem(qbn, mp.stages, false, u8);
    {
      ProfScope ps(ctx, SB_PROF_DENSE_SCAN, st);
      rc = u8 ? dispatch_mma<false, false, SB_STORAGE_U8, true>(qbn, tm_rows, tm_q, mp, grid, smem, st)
              : dispatch_mma<false, false, SB_STORAGE_F16, true>(qbn, tm_rows, tm_q, mp, grid, smem, st);
      if (rc) return rc;
    }
    RecoCombineParams cp;
    cp.keys = keys;
    cp.ld = n_pad;
    cp.n = ix.n;
    cp.e0 = e0;
    cp.r0 = r0;
    cp.req = req_d;
    cp.cd = cd;
    cp.mask = mask;
    cp.mask_qs = qs;
    cp.lo = lo;
    cp.hi = hi;
    dense_reco_combine_kernel<<<dim3((unsigned)((ix.n + 255) / 256), (unsigned)nr), 256, 0, st>>>(cp);
    RecoSelectParams sp;
    sp.lo = lo;
    sp.hi = hi;
    sp.ld = n_pad;
    sp.n = ix.n;
    sp.r0 = r0;
    sp.req = req_d;
    sp.ex = ex_pad;
    sp.qn = qn;
    sp.ex_fb = ex_fb;
    sp.slot = slot_view(ix);
    sp.k = k;
    sp.fallback = fb;
    sp.out_ids = out_ids;
    sp.out_scores = out_scores;
    sp.out_counts = out_counts;
    sp.mask = mask;
    sp.mask_qs = qs;
    sp.counter = ctx->fb_count_dev.as<unsigned long long>();
    {
      ProfScope ps(ctx, SB_PROF_DENSE_MERGE, st, 2);
      sel_kern<<<nr, kRecoThreads, 0, st>>>(sp);
      fb_kern<<<nr, kRecoThreads, 0, st>>>(sp);
    }
    SB_CUDA(cudaGetLastError());
    ctx->launches += 1;   // the combine
    r0 = r1;
  }
  return SB_OK;
}
