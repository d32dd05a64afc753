// dense_common.cuh -- pieces shared by the CUDA-core scan (dense.cu) and the wgmma batched scan (dense_mma.cu).
#pragma once
#include "common.cuh"

// What the exact stage (window re-score, brute-force fallback, filtered gather) reads of a slot.
struct SlotView {
  const __half* rows;   // [rows][d_pad] fp16 (float16 and float32 storage)
  const float* rows32;  // float32 storage: [rows][d_pad] the caller's x (read by the F32 instantiations only)
  const uint8_t* rows8; // uint8 storage: [rows][d_pad] the caller's x (read by the U8 instantiations only)
  const double* cfac;   // [rows] c of v = c * y (Dot / Euclid)
  int32_t metric;       // SB_METRIC_*
  int32_t d_pad;
  int32_t ch;           // d_pad / 8: eight-element chunks per row
  int64_t id_base;
};

inline SlotView slot_view(const DenseIndex& ix) {
  return {ix.rows, ix.rows32, ix.rows8, ix.cfac, ix.metric, ix.d_pad, ix.d_pad / 8, ix.id_base};
}

struct RescoreArgs {
  SlotView s;
  const float* q;       // this query's fp32 vector [d_pad]
  int32_t k;
  int64_t* out_ids;     // [k] of this query
  double* out_scores;   // [k]
  int32_t* out_count;   // [1]
};

// ---- approximate -> exact hand-off (DESIGN.md "K1: exactness") --------------------------------------------------------
// Both scans rank rows by an APPROXIMATE cosine a(x) (fp32 accumulation; the wgmma scan additionally rounds the
// normalised query to fp16).  With |a(x) - cos(x)| <= eps for every row, the exact top-k is contained in
//     W = { x : a(x) >= a_k - 2*eps },   a_k = the k-th largest approximate score
// (the k best approximate rows have cos >= a_k - eps, so the k-th best exact cosine is >= a_k - eps, and a row with
// cos >= a_k - eps has a >= a_k - 2*eps).  Every member of W is re-scored in fp64; W has no fixed size.  eps == 0
// (the all-zero query: every product is exactly 0) degenerates to "the k largest composite keys".
// A query whose window does not fit the shared-memory winner buffer -- or, in the CUDA-core scan, reaches the end of a
// full per-CTA list -- raises its fallback flag and is answered by dense_exact_fallback_kernel (brute force in fp64).

// eps of the CUDA-core scan: fp32 FMA chains over d_pad products of |x||q| <= 1 (normalised operands): gamma_d <= d*2^-24;
// doubled, plus 2^-19 for the fp32 normalisation of the query, the fp32 inverse row norm and the final product.
__host__ __device__ __forceinline__ float dense_eps_fp32(int d_pad) { return (float)d_pad * 1.1920929e-7f + 1.9073486e-6f; }
// accumulation part of the wgmma scan's eps: the tensor core's fp32 accumulator may truncate (<= 2 ulp per step)
__host__ __device__ __forceinline__ float dense_eps_mma_acc(int d_pad) { return (float)d_pad * 2.3841858e-7f + 1.9073486e-6f; }

// uint8 scan (DESIGN.md K1i): natural column c (0..63) of a 64-column block -> its column in the permuted fp16 query block.
// Byte c = 16 t + 4 s + j of a corpus row is the wgmma A element of k16 step s at k = 2 t + j (j < 2) or 2 t + 8 + j - 2
// (j >= 2) for the thread with lane % 4 = t, so the query's column c goes to 16 s + that k.
__host__ __device__ __forceinline__ int u8_query_column(int c) {
  const int t = c >> 4, s = (c >> 2) & 3, j = c & 3;
  return 16 * s + 2 * t + (j < 2 ? j : 6 + j);
}

// lower edge of the window as a composite key (keys >= it are members)
__device__ __forceinline__ unsigned long long window_lo_key(unsigned long long kth_lb_key, float eps) {
  if (!(eps > 0.f)) return kth_lb_key;
  const float lo = __fsub_rd(key32_score(kth_lb_key), __fmul_ru(2.f, eps));
  return (unsigned long long)f32_orderable(lo) << 32;
}

// Exact fp64 cosine of stored row `idx` with the fp32 query q (norm qn), computed by one full warp; every lane returns it.
__device__ __forceinline__ double exact_cosine_warp(const __half* rows, uint32_t idx, const float* q, int d_pad, int nch,
                                                    double qn, int lane) {
  const uint4* row = reinterpret_cast<const uint4*>(rows + (size_t)idx * d_pad);
  double dot = 0.0, xx = 0.0;
  for (int ch = lane; ch < nch; ch += 32) {
    const uint4 raw = __ldg(row + ch);
    const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
    const float4 qa = *reinterpret_cast<const float4*>(q + (size_t)ch * 8);
    const float4 qb = *reinterpret_cast<const float4*>(q + (size_t)ch * 8 + 4);
    const float qv[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 xf = __half22float2(h2[e]);
      const double x0 = (double)xf.x, x1 = (double)xf.y;
      dot = __fma_rn(x0, (double)qv[2 * e], dot);       // explicit FMAs: the one- and two-row variants must agree bit for bit
      dot = __fma_rn(x1, (double)qv[2 * e + 1], dot);
      xx = __fma_rn(x0, x0, xx);
      xx = __fma_rn(x1, x1, xx);
    }
  }
  for (int o = 16; o; o >>= 1) {
    dot += __shfl_xor_sync(0xffffffffu, dot, o);
    xx += __shfl_xor_sync(0xffffffffu, xx, o);
  }
  const double den = qn * sqrt(xx);
  return den > 0.0 ? dot / den : 0.0;
}

// ||q|| in fp64 (whole CTA; result broadcast through *qq_s)
__device__ __forceinline__ double query_norm_cta(const float* q, int d_pad, double* qq_s) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (warp == 0) {
    double s = 0.0;
    for (int i = lane; i < d_pad; i += 32) {
      const double v = (double)q[i];
      s += v * v;
    }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) *qq_s = s;
  }
  __syncthreads();
  return sqrt(*qq_s);
}

// (exact key desc, row asc) bitonic sort of P = 2^m (key, row) pairs in shared memory; (0, *) = empty sorts last
__device__ __forceinline__ void sort_exact_pairs(unsigned long long* ek, uint32_t* ei, int P, int tid, int nt) {
  for (int kk = 2; kk <= P; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += nt) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = ek[i], b = ek[ixj];
          const uint32_t ia = ei[i], ib = ei[ixj];
          const bool a_before_b = (a > b) || (a == b && ia < ib);
          const bool desc = (i & kk) == 0;
          if ((desc ? !a_before_b : a_before_b) && !(a == b && ia == ib)) {
            ek[i] = b; ek[ixj] = a;
            ei[i] = ib; ei[ixj] = ia;
          }
        }
      }
      __syncthreads();
    }
  }
}

// Exact fp64 ordering key of NR stored rows under Dot or Euclid (DESIGN.md K1e), one full warp; every lane returns them.
//   Dot:    c * sum q_i y_i                   (the score)
//   Euclid: -sqrt(sum (q_i - c y_i)^2)        (minus the distance: larger = better, like every other key; computed
//                                              directly, not as ||q||^2 - 2<q,v> + ||v||^2, which cancels when q ~ v)
// NR = 1 and NR = 2 perform the same operations in the same order per row, so they agree bit for bit.
template <int NR>
__device__ __forceinline__ void exact_metric_warp(int metric, const __half* rows, const double* cfac,
                                                  const uint32_t (&idx)[NR], const float* q, int d_pad, int nch,
                                                  int lane, double (&out)[NR]) {
  const bool euclid = metric == SB_METRIC_EUCLID;
  const uint4* r[NR];
  double c[NR], acc[NR];
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    r[i] = reinterpret_cast<const uint4*>(rows + (size_t)idx[i] * d_pad);
    c[i] = __ldg(cfac + idx[i]);
    acc[i] = 0.0;
  }
  for (int ch = lane; ch < nch; ch += 32) {
    const float4 qa = *reinterpret_cast<const float4*>(q + (size_t)ch * 8);
    const float4 qb = *reinterpret_cast<const float4*>(q + (size_t)ch * 8 + 4);
    const float qv[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
    uint4 raw[NR];
#pragma unroll
    for (int i = 0; i < NR; ++i) raw[i] = __ldg(r[i] + ch);
#pragma unroll
    for (int i = 0; i < NR; ++i) {
      const __half2* h2 = reinterpret_cast<const __half2*>(&raw[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 xf = __half22float2(h2[e]);
        const double x0 = (double)xf.x, x1 = (double)xf.y;
        if (euclid) {
          const double t0 = __fma_rn(-c[i], x0, (double)qv[2 * e]);
          const double t1 = __fma_rn(-c[i], x1, (double)qv[2 * e + 1]);
          acc[i] = __fma_rn(t0, t0, acc[i]);
          acc[i] = __fma_rn(t1, t1, acc[i]);
        } else {
          acc[i] = __fma_rn(x0, (double)qv[2 * e], acc[i]);
          acc[i] = __fma_rn(x1, (double)qv[2 * e + 1], acc[i]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    for (int o = 16; o; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
    out[i] = euclid ? -sqrt(acc[i]) : c[i] * acc[i];
  }
}

// Exact fp64 ordering key of NR float32-storage rows x (DESIGN.md K1g), one full warp; every lane returns them.
//   Cosine: <q, x> / (||q|| ||x||)   (0 for a zero row or query; qn = ||q||)
//   Dot:    <q, x>
//   Euclid: -sqrt(sum (q_i - x_i)^2)  (computed directly: q = x gives exactly 0)
// Lane l reads 8 floats of chunk c = l + 32 j of every row with two float4 loads (rows are 32-byte aligned).  NR = 1 and
// NR = 2 perform the same operations in the same order per row, so they agree bit for bit.
template <int NR>
__device__ __forceinline__ void exact_f32_warp(int metric, const float* rows32, const uint32_t (&idx)[NR], const float* q,
                                               int d_pad, int nch, double qn, int lane, double (&out)[NR]) {
  const bool euclid = metric == SB_METRIC_EUCLID, cosine = metric == SB_METRIC_COSINE;
  const float4* r[NR];
  double acc[NR], xx[NR];
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    r[i] = reinterpret_cast<const float4*>(rows32 + (size_t)idx[i] * d_pad);
    acc[i] = 0.0;
    xx[i] = 0.0;
  }
  for (int ch = lane; ch < nch; ch += 32) {
    const float4 qa = *reinterpret_cast<const float4*>(q + (size_t)ch * 8);
    const float4 qb = *reinterpret_cast<const float4*>(q + (size_t)ch * 8 + 4);
    const float qv[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
    float4 raw[NR][2];
#pragma unroll
    for (int i = 0; i < NR; ++i) {
      raw[i][0] = __ldg(r[i] + 2 * ch);
      raw[i][1] = __ldg(r[i] + 2 * ch + 1);
    }
#pragma unroll
    for (int i = 0; i < NR; ++i) {
      const float xv[8] = {raw[i][0].x, raw[i][0].y, raw[i][0].z, raw[i][0].w,
                           raw[i][1].x, raw[i][1].y, raw[i][1].z, raw[i][1].w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const double x = (double)xv[e], qe = (double)qv[e];
        if (euclid) {
          const double t = __dsub_rn(qe, x);
          acc[i] = __fma_rn(t, t, acc[i]);
        } else {
          acc[i] = __fma_rn(x, qe, acc[i]);
          if (cosine) xx[i] = __fma_rn(x, x, xx[i]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    for (int o = 16; o; o >>= 1) {
      acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
      xx[i] += __shfl_xor_sync(0xffffffffu, xx[i], o);
    }
    if (euclid) {
      out[i] = -sqrt(acc[i]);
    } else if (cosine) {
      const double den = qn * sqrt(xx[i]);
      out[i] = den > 0.0 ? acc[i] / den : 0.0;
    } else {
      out[i] = acc[i];
    }
  }
}

// Exact fp64 ordering key of NR uint8-storage rows x (DESIGN.md K1i), one full warp; every lane returns them.  The same
// formulas and operation order as exact_f32_warp; every product q_i x_i and every x_i^2 is exact in fp64.  Lane l reads
// the 8 bytes of chunk c = l + 32 j of every row with one 8-byte load (rows are 64-byte aligned).
template <int NR>
__device__ __forceinline__ void exact_u8_warp(int metric, const uint8_t* rows8, const uint32_t (&idx)[NR], const float* q,
                                              int d_pad, int nch, double qn, int lane, double (&out)[NR]) {
  const bool euclid = metric == SB_METRIC_EUCLID, cosine = metric == SB_METRIC_COSINE;
  const uint2* r[NR];
  double acc[NR], xx[NR];
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    r[i] = reinterpret_cast<const uint2*>(rows8 + (size_t)idx[i] * d_pad);
    acc[i] = 0.0;
    xx[i] = 0.0;
  }
  for (int ch = lane; ch < nch; ch += 32) {
    const float4 qa = *reinterpret_cast<const float4*>(q + (size_t)ch * 8);
    const float4 qb = *reinterpret_cast<const float4*>(q + (size_t)ch * 8 + 4);
    const float qv[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
    uint2 raw[NR];
#pragma unroll
    for (int i = 0; i < NR; ++i) raw[i] = __ldg(r[i] + ch);
#pragma unroll
    for (int i = 0; i < NR; ++i) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t w = e < 4 ? raw[i].x : raw[i].y;
        const double x = (double)((w >> (8 * (e & 3))) & 0xffu), qe = (double)qv[e];
        if (euclid) {
          const double t = __dsub_rn(qe, x);
          acc[i] = __fma_rn(t, t, acc[i]);
        } else {
          acc[i] = __fma_rn(x, qe, acc[i]);
          if (cosine) xx[i] = __fma_rn(x, x, xx[i]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    for (int o = 16; o; o >>= 1) {
      acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
      xx[i] += __shfl_xor_sync(0xffffffffu, xx[i], o);
    }
    if (euclid) {
      out[i] = -sqrt(acc[i]);
    } else if (cosine) {
      const double den = qn * sqrt(xx[i]);
      out[i] = den > 0.0 ? acc[i] / den : 0.0;
    } else {
      out[i] = acc[i];
    }
  }
}

// exact ordering key of one stored row under the slot's metric (Cosine: the existing cosine path)
__device__ __forceinline__ double exact_key_warp(int metric, const __half* rows, const double* cfac, uint32_t idx,
                                                 const float* q, int d_pad, int nch, double qn, int lane) {
  if (metric == SB_METRIC_COSINE) return exact_cosine_warp(rows, idx, q, d_pad, nch, qn, lane);
  const uint32_t ix[1] = {idx};
  double s[1];
  exact_metric_warp<1>(metric, rows, cfac, ix, q, d_pad, nch, lane, s);
  return s[0];
}

// exact ordering key of one row under the slot's storage ST (SB_STORAGE_*): float32 and uint8 score the caller's x,
// float16 the stored fp16 representation
template <int ST>
__device__ __forceinline__ double exact_key_row(const SlotView& v, uint32_t idx, const float* q, double qn, int lane) {
  if constexpr (ST == SB_STORAGE_F32) {
    const uint32_t ix[1] = {idx};
    double s[1];
    exact_f32_warp<1>(v.metric, v.rows32, ix, q, v.d_pad, v.ch, qn, lane, s);
    return s[0];
  } else if constexpr (ST == SB_STORAGE_U8) {
    const uint32_t ix[1] = {idx};
    double s[1];
    exact_u8_warp<1>(v.metric, v.rows8, ix, q, v.d_pad, v.ch, qn, lane, s);
    return s[0];
  } else {
    return exact_key_warp(v.metric, v.rows, v.cfac, idx, q, v.d_pad, v.ch, qn, lane);
  }
}

// first min(k, P) sorted pairs -> this query's output rows (Euclid keys are minus the distance: the score is the distance)
__device__ __forceinline__ void emit_exact_pairs(const unsigned long long* ek, const uint32_t* ei, int P,
                                                 const RescoreArgs& p) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const bool euclid = p.s.metric == SB_METRIC_EUCLID;
  for (int i = tid; i < p.k; i += nt) {
    const bool valid = (i < P) && ek[i] != 0ull;
    p.out_ids[i] = valid ? p.s.id_base + (int64_t)ei[i] : -1;
    double s = 0.0;
    if (valid) s = euclid ? -orderable_f64(ek[i]) : orderable_f64(ek[i]);
    p.out_scores[i] = s;
  }
  if (tid == 0) {
    int lo = 0, hi = min(p.k, P);  // valid entries are a prefix (empty keys sort last)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ek[mid] != 0ull) lo = mid + 1; else hi = mid;
    }
    p.out_count[0] = lo;
  }
}

// Two rows at once (twice the loads in flight per warp): same arithmetic and order as exact_cosine_warp, per row.
__device__ __forceinline__ void exact_cosine_warp2(const __half* rows, uint32_t idx0, uint32_t idx1, const float* q, int d_pad,
                                                   int nch, double qn, int lane, double* out0, double* out1) {
  const uint4* r0 = reinterpret_cast<const uint4*>(rows + (size_t)idx0 * d_pad);
  const uint4* r1 = reinterpret_cast<const uint4*>(rows + (size_t)idx1 * d_pad);
  double dot0 = 0.0, xx0 = 0.0, dot1 = 0.0, xx1 = 0.0;
  for (int ch = lane; ch < nch; ch += 32) {
    const uint4 raw0 = __ldg(r0 + ch), raw1 = __ldg(r1 + ch);
    const __half2* h0 = reinterpret_cast<const __half2*>(&raw0);
    const __half2* h1 = reinterpret_cast<const __half2*>(&raw1);
    const float4 qa = *reinterpret_cast<const float4*>(q + (size_t)ch * 8);
    const float4 qb = *reinterpret_cast<const float4*>(q + (size_t)ch * 8 + 4);
    const float qv[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 a = __half22float2(h0[e]), b = __half22float2(h1[e]);
      const double a0 = (double)a.x, a1 = (double)a.y, b0 = (double)b.x, b1 = (double)b.y;
      dot0 = __fma_rn(a0, (double)qv[2 * e], dot0);
      dot0 = __fma_rn(a1, (double)qv[2 * e + 1], dot0);
      xx0 = __fma_rn(a0, a0, xx0);
      xx0 = __fma_rn(a1, a1, xx0);
      dot1 = __fma_rn(b0, (double)qv[2 * e], dot1);
      dot1 = __fma_rn(b1, (double)qv[2 * e + 1], dot1);
      xx1 = __fma_rn(b0, b0, xx1);
      xx1 = __fma_rn(b1, b1, xx1);
    }
  }
  for (int o = 16; o; o >>= 1) {
    dot0 += __shfl_xor_sync(0xffffffffu, dot0, o);
    xx0 += __shfl_xor_sync(0xffffffffu, xx0, o);
    dot1 += __shfl_xor_sync(0xffffffffu, dot1, o);
    xx1 += __shfl_xor_sync(0xffffffffu, xx1, o);
  }
  const double den0 = qn * sqrt(xx0), den1 = qn * sqrt(xx1);
  *out0 = den0 > 0.0 ? dot0 / den0 : 0.0;
  *out1 = den1 > 0.0 ? dot1 / den1 : 0.0;
}

// Exact fp64 re-score of the window members sel[0..nsel) (composite keys) against the STORED fp16 rows and the fp32
// query, final order (score desc, row asc), emit k results.  Whole-CTA cooperative; ek/ei are P-entry shared-memory
// arrays (P = power of two >= nsel), qq_s a shared double, q_s a shared-memory staging area for the query (d_pad floats;
// the L2 round trip of the query per re-scored row was a third of the stage's latency).  ST = SB_STORAGE_F32 / _U8: the
// window is re-scored against the caller's rows (exact_f32_warp / exact_u8_warp).
template <int ST>
__device__ __forceinline__ void rescore_and_emit(const unsigned long long* sel, int nsel, int P, unsigned long long* ek,
                                                 uint32_t* ei, double* qq_s_ptr, float* q_s, const RescoreArgs p) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x, nw = nt >> 5;
  const SlotView& v = p.s;
  for (int i = tid; i < v.d_pad; i += nt) q_s[i] = p.q[i];
  __syncthreads();
  const double qn = query_norm_cta(q_s, v.d_pad, qq_s_ptr);
  for (int c = warp; c < P; c += 2 * nw) {
    const int c1 = c + nw;
    const unsigned long long key0 = c < nsel ? sel[c] : 0ull;
    const unsigned long long key1 = (c1 < P && c1 < nsel) ? sel[c1] : 0ull;
    unsigned long long o0 = 0ull, o1 = 0ull;
    uint32_t i0 = 0xffffffffu, i1 = 0xffffffffu;
    if (key0 != 0ull && key1 != 0ull) {
      i0 = key32_idx(key0);
      i1 = key32_idx(key1);
      double s0, s1;
      if constexpr (ST == SB_STORAGE_F32) {
        const uint32_t ix[2] = {i0, i1};
        double s[2];
        exact_f32_warp<2>(v.metric, v.rows32, ix, q_s, v.d_pad, v.ch, qn, lane, s);
        s0 = s[0];
        s1 = s[1];
      } else if constexpr (ST == SB_STORAGE_U8) {
        const uint32_t ix[2] = {i0, i1};
        double s[2];
        exact_u8_warp<2>(v.metric, v.rows8, ix, q_s, v.d_pad, v.ch, qn, lane, s);
        s0 = s[0];
        s1 = s[1];
      } else if (v.metric == SB_METRIC_COSINE) {
        exact_cosine_warp2(v.rows, i0, i1, q_s, v.d_pad, v.ch, qn, lane, &s0, &s1);
      } else {
        const uint32_t ix[2] = {i0, i1};
        double s[2];
        exact_metric_warp<2>(v.metric, v.rows, v.cfac, ix, q_s, v.d_pad, v.ch, lane, s);
        s0 = s[0];
        s1 = s[1];
      }
      o0 = f64_orderable(s0);
      o1 = f64_orderable(s1);
    } else if (key0 != 0ull) {
      i0 = key32_idx(key0);
      o0 = f64_orderable(exact_key_row<ST>(v, i0, q_s, qn, lane));
    } else if (key1 != 0ull) {
      i1 = key32_idx(key1);
      o1 = f64_orderable(exact_key_row<ST>(v, i1, q_s, qn, lane));
    }
    if (key0 != 0ull && o0 == 0ull) o0 = 1ull;  // keep 0 reserved for "empty"
    if (key1 != 0ull && o1 == 0ull) o1 = 1ull;
    if (lane == 0) {
      ek[c] = o0;
      ei[c] = i0;
      if (c1 < P) {
        ek[c1] = o1;
        ei[c1] = i1;
      }
    }
  }
  __syncthreads();
  sort_exact_pairs(ek, ei, P, tid, nt);
  emit_exact_pairs(ek, ei, P, p);
}
