// fuse.cu -- K3: rank / score fusion (rrf, weighted_rrf, comb_sum) + additive scorer signals + stable ranking,
//            and K6: merge of all-gathered per-shard top-k lists.
//
// Replaces the fusion block of HybridRetriever.retrieve (reference src/core/retrievers/hybrid.py:204-298).
// One CTA per query; everything lives in shared memory (<= a few thousand candidates) -- latency bound, not HBM bound.
//
// Exact Python semantics reproduced (fp64, explicit _rn intrinsics, no contraction):
//   * `fused_scores` is a defaultdict(float): insertion order = first occurrence in dense ++ sparse ++ plugin order,
//     and every `+=` happens in that same traversal order (hybrid.py:222-259).
//   * rrf / weighted_rrf: EVERY occurrence contributes w * (1.0 / (rrf_k + rank)), rank 0-based inside its own list.
//   * comb_sum: per list a dict id -> LAST raw score, min-max normalised over the dict values (all equal -> 1.0),
//     one contribution per unique id, weights dense_weight / sparse_weight / 0.2 (hybrid.py:211-220,229-259).
//   * scorer-plugin scores are added one plugin at a time to the merged documents
//     (unique dense ids, then sparse-only ids; hybrid.py:262-285).
//   * sorted(..., reverse=True) is stable -> order = (score desc, insertion index asc); truncate to k.
#include <algorithm>
#include <string.h>

#include "common.cuh"

namespace {

constexpr int kFuseThreads = 256;

struct FuseParams {
  int method;
  double rrf_k, w_dense, w_sparse;
  const int64_t *d_ids, *s_ids, *p_ids;
  const double *d_sc, *s_sc, *p_sc;
  const int32_t *d_n, *s_n, *p_n;
  int d_stride, s_stride, p_stride;
  const double* extra;  // [B][n_extra][e_stride] or NULL
  int n_extra, e_stride;
  int k;
  int m_max;  // smem capacity in items
  int64_t* out_ids;
  double* out_scores;
  int32_t* out_src;
  int32_t* out_counts;
};

__global__ void __launch_bounds__(kFuseThreads) fuse_kernel(const FuseParams p) {
  extern __shared__ __align__(16) uint8_t fsm[];
  const int tid = threadIdx.x, qi = blockIdx.x;
  const int nd = p.d_ids ? min(p.d_n[qi], p.d_stride) : 0;
  const int ns = p.s_ids ? min(p.s_n[qi], p.s_stride) : 0;
  const int np = p.p_ids ? min(p.p_n[qi], p.p_stride) : 0;
  const int M = nd + ns + np;
  int64_t* ids = reinterpret_cast<int64_t*>(fsm);                   // [m_max]
  double* raw = reinterpret_cast<double*>(ids + p.m_max);           // [m_max] raw score -> contribution
  double* fused = raw + p.m_max;                                    // [m_max] valid at representative slots
  int32_t* first = reinterpret_cast<int32_t*>(fused + p.m_max);     // [m_max] first occurrence (global)
  int32_t* order = first + p.m_max;                                 // [m_max] insertion order of representatives
  __shared__ double s_min[3], s_max[3];
  __shared__ int s_nrep;

  for (int t = tid; t < M; t += kFuseThreads) {
    if (t < nd) {
      ids[t] = p.d_ids[(size_t)qi * p.d_stride + t];
      raw[t] = p.d_sc[(size_t)qi * p.d_stride + t];
    } else if (t < nd + ns) {
      ids[t] = p.s_ids[(size_t)qi * p.s_stride + (t - nd)];
      raw[t] = p.s_sc[(size_t)qi * p.s_stride + (t - nd)];
    } else {
      ids[t] = p.p_ids[(size_t)qi * p.p_stride + (t - nd - ns)];
      raw[t] = p.p_sc[(size_t)qi * p.p_stride + (t - nd - ns)];
    }
  }
  __syncthreads();
  // first occurrence of every id in concatenation order
  for (int t = tid; t < M; t += kFuseThreads) {
    const int64_t id = ids[t];
    int f = t;
    for (int u = 0; u < t; ++u) {
      if (ids[u] == id) {
        f = u;
        break;
      }
    }
    first[t] = f;
  }
  __syncthreads();

  const int lo[3] = {0, nd, nd + ns}, hi[3] = {nd, nd + ns, M};
  if (p.method == SB_FUSE_COMB_SUM) {
    // dict semantics per list: value of an id = raw of its LAST occurrence inside the list, kept at the FIRST slot
    for (int t = tid; t < M; t += kFuseThreads) {
      const int L = t < nd ? 0 : (t < nd + ns ? 1 : 2);
      const int64_t id = ids[t];
      bool is_first = true;
      for (int u = lo[L]; u < t; ++u)
        if (ids[u] == id) {
          is_first = false;
          break;
        }
      double v = raw[t];
      if (is_first) {
        for (int u = t + 1; u < hi[L]; ++u)
          if (ids[u] == id) v = raw[u];
      }
      // stash: fused[] temporarily holds the dict value, order[] the is-first flag
      fused[t] = v;
      order[t] = is_first ? 1 : 0;
    }
    __syncthreads();
    if (tid < 3) {
      double mn = 0.0, mx = 0.0;
      bool any = false;
      for (int t = lo[tid]; t < hi[tid]; ++t) {
        if (!order[t]) continue;
        const double v = fused[t];
        if (!any) {
          mn = mx = v;
          any = true;
        } else {
          if (v < mn) mn = v;
          if (v > mx) mx = v;
        }
      }
      s_min[tid] = mn;
      s_max[tid] = mx;
    }
    __syncthreads();
    for (int t = tid; t < M; t += kFuseThreads) {
      const int L = t < nd ? 0 : (t < nd + ns ? 1 : 2);
      double c = 0.0;
      bool contributes = order[t] != 0;
      if (contributes) {
        const double mn = s_min[L], mx = s_max[L];
        double nscore;
        if (mx <= mn) {
          nscore = 1.0;
        } else {
          nscore = __ddiv_rn(__dsub_rn(fused[t], mn), __dsub_rn(mx, mn));
        }
        const double w = L == 0 ? p.w_dense : (L == 1 ? p.w_sparse : 0.2);
        c = __dmul_rn(w, nscore);
      }
      raw[t] = c;
      first[t] = contributes ? first[t] : -1 - first[t];  // negative = occurrence that adds nothing
    }
    __syncthreads();
  } else {
    for (int t = tid; t < M; t += kFuseThreads) {
      const int L = t < nd ? 0 : (t < nd + ns ? 1 : 2);
      const int rank = t - lo[L];
      const double inv = __ddiv_rn(1.0, __dadd_rn(p.rrf_k, (double)rank));
      double w = 1.0;
      if (p.method == SB_FUSE_WEIGHTED_RRF && L < 2) w = L == 0 ? p.w_dense : p.w_sparse;
      raw[t] = __dmul_rn(w, inv);
    }
    __syncthreads();
  }

  // representatives + insertion order
  if (tid == 0) {
    int r = 0;
    for (int t = 0; t < M; ++t) {
      const int f = first[t] < 0 ? -1 - first[t] : first[t];
      if (f == t) order[t] = r++;
      else order[t] = -1;
    }
    s_nrep = r;
  }
  __syncthreads();
  const int nrep = s_nrep;
  // sequential accumulation per representative, in traversal order
  for (int u = tid; u < M; u += kFuseThreads) {
    if (order[u] < 0) continue;
    double acc = 0.0;
    for (int t = u; t < M; ++t) {
      const int ft = first[t];
      if (ft == u) acc = __dadd_rn(acc, raw[t]);
    }
    // scorer-plugin signals for merged documents (representatives that own a dense or sparse document)
    if (p.extra && u < nd + ns) {
      const int m = order[u];
      if (m < p.e_stride) {
        for (int e = 0; e < p.n_extra; ++e)
          acc = __dadd_rn(acc, p.extra[((size_t)qi * p.n_extra + e) * p.e_stride + m]);
      }
    }
    fused[u] = acc;
  }
  __syncthreads();
  // stable descending rank among representatives
  for (int u = tid; u < M; u += kFuseThreads) {
    if (order[u] < 0) continue;
    const double su = fused[u];
    int pos = 0;
    for (int v = 0; v < M; ++v) {
      if (order[v] < 0 || v == u) continue;
      const double sv = fused[v];
      if (sv > su || (sv == su && v < u)) ++pos;
    }
    if (pos < p.k) {
      int src = 0;
      const int64_t id = ids[u];
      if (u < nd) src |= 1;
      for (int t = nd; t < nd + ns; ++t)
        if (ids[t] == id) {
          src |= 2;
          break;
        }
      p.out_ids[(size_t)qi * p.k + pos] = id;
      p.out_scores[(size_t)qi * p.k + pos] = su;
      p.out_src[(size_t)qi * p.k + pos] = src;
    }
  }
  const int cnt = min(nrep, p.k);
  for (int i = cnt + tid; i < p.k; i += kFuseThreads) {
    p.out_ids[(size_t)qi * p.k + i] = -1;
    p.out_scores[(size_t)qi * p.k + i] = 0.0;
    p.out_src[(size_t)qi * p.k + i] = 0;
  }
  if (tid == 0) p.out_counts[qi] = cnt;
}

// ------------------------------------------------------------------------------------------------ K6 shard merge
// shard g's ids [B][k] / scores [B][k] / counts [B] start shard_stride_bytes * g after the base pointers (the layout
// of one all-gathered record buffer) -> global top-k per query by (score desc, id asc).
__global__ void __launch_bounds__(256) merge_shards_kernel(const int64_t* in_ids0, const double* in_scores0,
                                                           const int32_t* in_counts0, int64_t shard_stride_bytes,
                                                           int G, int B, int k, int len_pow2, int64_t* out_ids,
                                                           double* out_scores, int32_t* out_counts) {
  extern __shared__ __align__(16) uint8_t msm[];
  unsigned long long* key = reinterpret_cast<unsigned long long*>(msm);
  int64_t* ids = reinterpret_cast<int64_t*>(key + len_pow2);
  const int tid = threadIdx.x, qi = blockIdx.x;
  for (int i = tid; i < len_pow2; i += blockDim.x) {
    unsigned long long kk = 0ull;
    int64_t id = 0x7fffffffffffffffll;
    if (i < G * k) {
      const int g = i / k, r = i - g * k;
      const size_t sh = (size_t)g * (size_t)shard_stride_bytes;
      const int32_t* in_counts = reinterpret_cast<const int32_t*>(reinterpret_cast<const char*>(in_counts0) + sh);
      if (r < in_counts[qi]) {
        const double* in_scores = reinterpret_cast<const double*>(reinterpret_cast<const char*>(in_scores0) + sh);
        const int64_t* in_ids = reinterpret_cast<const int64_t*>(reinterpret_cast<const char*>(in_ids0) + sh);
        kk = f64_orderable(in_scores[(size_t)qi * k + r]);
        if (kk == 0ull) kk = 1ull;
        id = in_ids[(size_t)qi * k + r];
      }
    }
    key[i] = kk;
    ids[i] = id;
  }
  __syncthreads();
  for (int kk = 2; kk <= len_pow2; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < len_pow2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = key[i], b = key[ixj];
          const int64_t ia = ids[i], ib = ids[ixj];
          const bool a_first = (a > b) || (a == b && ia < ib);
          const bool desc = (i & kk) == 0;
          if ((desc ? !a_first : a_first) && !(a == b && ia == ib)) {
            key[i] = b; key[ixj] = a;
            ids[i] = ib; ids[ixj] = ia;
          }
        }
      }
      __syncthreads();
    }
  }
  int cnt = 0;
  for (int i = tid; i < k; i += blockDim.x) {
    const bool valid = i < len_pow2 && key[i] != 0ull;
    out_ids[(size_t)qi * k + i] = valid ? ids[i] : -1;
    out_scores[(size_t)qi * k + i] = valid ? orderable_f64(key[i]) : 0.0;
  }
  if (tid == 0) {
    int lo = 0, hi = min(k, len_pow2);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (key[mid] != 0ull) lo = mid + 1; else hi = mid;
    }
    cnt = lo;
    out_counts[qi] = cnt;
  }
}

// ------------------------------------------------------------------------------------------------ K7: document selector
// Batched form of select_documents_node (reference src/core/graph/nodes.py:272-337): per query, stable sort of the candidates
// by score (desc), ids seen before are dropped, the first top_k unique documents are walked, blank documents (0 chars) are
// skipped, a document is kept while the running len(text) // 4 estimate stays <= max_tokens and the first one that does
// not fit ends the walk.  One CTA per query; the walk itself is sequential by definition (<= top_k steps, one thread).
template <typename ScoreT>
__global__ void __launch_bounds__(128) select_docs_kernel(const int64_t* __restrict__ cand_ids,
                                                          const ScoreT* __restrict__ cand_scores,
                                                          const int32_t* __restrict__ cand_cnt, int k, int top_k,
                                                          int max_tokens, const int32_t* __restrict__ doc_chars,
                                                          int64_t n_docs, int64_t id_base, int64_t* __restrict__ out_ids,
                                                          ScoreT* __restrict__ out_scores, int32_t* __restrict__ out_counts,
                                                          int32_t* __restrict__ out_tokens) {
  extern __shared__ __align__(16) uint8_t sel_sm[];
  double* sc = reinterpret_cast<double*>(sel_sm);        // [k]
  int32_t* order = reinterpret_cast<int32_t*>(sc + k);   // [k] candidate index at every sorted position
  const int b = blockIdx.x, n = min(max(cand_cnt[b], 0), k);
  for (int j = threadIdx.x; j < n; j += blockDim.x) sc[j] = (double)cand_scores[(size_t)b * k + j];
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const double s = sc[j];
    int pos = 0;
    for (int i = 0; i < n; ++i) pos += (sc[i] > s) || (sc[i] == s && i < j);  // sorted(..., reverse=True) is stable
    order[pos] = j;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int64_t* ids = cand_ids + (size_t)b * k;
  int uniq = 0, nsel = 0, total = 0;
  for (int p = 0; p < n && uniq < top_k; ++p) {
    const int j = order[p];
    const int64_t id = ids[j];
    bool seen = false;
    for (int q = 0; q < p && !seen; ++q) seen = ids[order[q]] == id;
    if (seen) continue;
    ++uniq;
    const int64_t row = id - id_base;
    const int chars = (row >= 0 && row < n_docs) ? doc_chars[row] : 0;
    if (chars <= 0) continue;  // blank document
    const int tok = chars / 4;
    if (total + tok > max_tokens) break;
    out_ids[(size_t)b * top_k + nsel] = id;
    out_scores[(size_t)b * top_k + nsel] = cand_scores[(size_t)b * k + j];
    ++nsel;
    total += tok;
  }
  for (int q = nsel; q < top_k; ++q) {
    out_ids[(size_t)b * top_k + q] = -1;
    out_scores[(size_t)b * top_k + q] = (ScoreT)0;
  }
  out_counts[b] = nsel;
  out_tokens[b] = total;
}


}  // namespace

int sb_fuse_enqueue(sb_ctx* ctx, int32_t method, double rrf_k, double w_dense, double w_sparse, int32_t B,
                    const int64_t* d_ids, const double* d_sc, const int32_t* d_n, int32_t d_stride,
                    const int64_t* s_ids, const double* s_sc, const int32_t* s_n, int32_t s_stride,
                    const int64_t* p_ids, const double* p_sc, const int32_t* p_n, int32_t p_stride,
                    const double* extra, int32_t n_extra, int32_t e_stride, int32_t k, int64_t* out_ids,
                    double* out_scores, int32_t* out_src, int32_t* out_counts, cudaStream_t st) {
  SB_REQUIRE(method >= SB_FUSE_RRF && method <= SB_FUSE_COMB_SUM, SB_ERR_ARG, "sb_fuse: unknown fusion method %d",
             method);
  const int m_max = (d_ids ? d_stride : 0) + (s_ids ? s_stride : 0) + (p_ids ? p_stride : 0);
  SB_REQUIRE(m_max <= 4096, SB_ERR_UNSUPPORTED, "sb_fuse: %d candidates per query exceed the 4096 limit", m_max);
  FuseParams fp;
  fp.method = method;
  fp.rrf_k = rrf_k;
  fp.w_dense = w_dense;
  fp.w_sparse = w_sparse;
  fp.d_ids = d_ids; fp.d_sc = d_sc; fp.d_n = d_n; fp.d_stride = d_stride;
  fp.s_ids = s_ids; fp.s_sc = s_sc; fp.s_n = s_n; fp.s_stride = s_stride;
  fp.p_ids = p_ids; fp.p_sc = p_sc; fp.p_n = p_n; fp.p_stride = p_stride;
  fp.extra = (extra && n_extra > 0) ? extra : nullptr;
  fp.n_extra = n_extra;
  fp.e_stride = e_stride;
  fp.k = k;
  fp.m_max = std::max(m_max, 1);
  fp.out_ids = out_ids;
  fp.out_scores = out_scores;
  fp.out_src = out_src;
  fp.out_counts = out_counts;
  const size_t smem = (size_t)fp.m_max * (8 + 8 + 8 + 4 + 4) + 16;
  SB_CUDA(cudaFuncSetAttribute(fuse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  {
    ProfScope ps(ctx, SB_PROF_FUSE, st);
    fuse_kernel<<<B, kFuseThreads, smem, st>>>(fp);
  }
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

extern "C" {

int sb_fuse_dev(sb_ctx* ctx, int32_t method, double rrf_k, double w_dense, double w_sparse, int32_t B,
                const int64_t* d_ids, const double* d_sc, const int32_t* d_n, int32_t d_stride, const int64_t* s_ids,
                const double* s_sc, const int32_t* s_n, int32_t s_stride, const int64_t* p_ids, const double* p_sc,
                const int32_t* p_n, int32_t p_stride, const double* extra, int32_t n_extra, int32_t e_stride,
                int32_t k, int64_t* out_ids, double* out_scores, int32_t* out_src, int32_t* out_counts, void* stream) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_fuse_dev: ctx is NULL");
  SB_REQUIRE(B >= 0 && k > 0, SB_ERR_ARG, "sb_fuse_dev: bad B=%d k=%d", B, k);
  if (B == 0) return SB_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  return sb_fuse_enqueue(ctx, method, rrf_k, w_dense, w_sparse, B, d_ids, d_sc, d_n, d_stride, s_ids, s_sc, s_n,
                         s_stride, p_ids, p_sc, p_n, p_stride, extra, n_extra, e_stride, k, out_ids, out_scores,
                         out_src, out_counts, pick_stream(ctx, stream));
}

int sb_fuse(sb_ctx* ctx, int32_t method, double rrf_k, double w_dense, double w_sparse, int32_t B,
            const int64_t* d_ids, const double* d_sc, const int32_t* d_n, int32_t d_stride, const int64_t* s_ids,
            const double* s_sc, const int32_t* s_n, int32_t s_stride, const int64_t* p_ids, const double* p_sc,
            const int32_t* p_n, int32_t p_stride, const double* extra, int32_t n_extra, int32_t e_stride, int32_t k,
            int64_t* out_ids, double* out_scores, int32_t* out_src, int32_t* out_counts) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_fuse: ctx is NULL");
  SB_REQUIRE(B >= 0 && k > 0, SB_ERR_ARG, "sb_fuse: bad B=%d k=%d", B, k);
  if (B == 0) return SB_OK;
  SB_REQUIRE(out_ids && out_scores && out_src && out_counts, SB_ERR_ARG, "sb_fuse: NULL output buffer");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = ctx->stream;
  // pack all inputs into one pinned staging buffer -> one H2D copy
  struct Seg { const void* src; size_t bytes; size_t off; };
  Seg seg[10];
  int nseg = 0;
  size_t total = 0;
  auto add = [&](const void* src, size_t bytes) -> size_t {
    if (!src || bytes == 0) return (size_t)-1;
    total = (total + 15) & ~(size_t)15;
    seg[nseg] = {src, bytes, total};
    total += bytes;
    return seg[nseg++].off;
  };
  const bool has_d = d_ids && d_stride > 0, has_s = s_ids && s_stride > 0, has_p = p_ids && p_stride > 0;
  const size_t o_di = has_d ? add(d_ids, (size_t)B * d_stride * 8) : (size_t)-1;
  const size_t o_ds = has_d ? add(d_sc, (size_t)B * d_stride * 8) : (size_t)-1;
  const size_t o_dn = has_d ? add(d_n, (size_t)B * 4) : (size_t)-1;
  const size_t o_si = has_s ? add(s_ids, (size_t)B * s_stride * 8) : (size_t)-1;
  const size_t o_ss = has_s ? add(s_sc, (size_t)B * s_stride * 8) : (size_t)-1;
  const size_t o_sn = has_s ? add(s_n, (size_t)B * 4) : (size_t)-1;
  const size_t o_pi = has_p ? add(p_ids, (size_t)B * p_stride * 8) : (size_t)-1;
  const size_t o_ps = has_p ? add(p_sc, (size_t)B * p_stride * 8) : (size_t)-1;
  const size_t o_pn = has_p ? add(p_n, (size_t)B * 4) : (size_t)-1;
  const bool has_e = extra && n_extra > 0 && e_stride > 0;
  const size_t o_ex = has_e ? add(extra, (size_t)B * n_extra * e_stride * 8) : (size_t)-1;
  SB_REQUIRE((!has_d || (d_sc && d_n)) && (!has_s || (s_sc && s_n)) && (!has_p || (p_sc && p_n)), SB_ERR_ARG,
             "sb_fuse: list given without scores/counts");
  int rc;
  if ((rc = ctx->pin_in.reserve(total + 16))) return rc;
  if ((rc = ctx->misc_dev.reserve(total + 16))) return rc;
  uint8_t* pi = ctx->pin_in.as<uint8_t>();
  for (int i = 0; i < nseg; ++i) memcpy(pi + seg[i].off, seg[i].src, seg[i].bytes);
  if (total) SB_CUDA(cudaMemcpyAsync(ctx->misc_dev.p, pi, total, cudaMemcpyHostToDevice, st));
  uint8_t* dv = ctx->misc_dev.as<uint8_t>();
  auto at = [&](size_t off) -> const void* { return off == (size_t)-1 ? nullptr : dv + off; };
  const size_t nid = (size_t)B * k;
  if ((rc = ctx->out_ids_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_sc_dev.reserve(nid * 8))) return rc;
  if ((rc = ctx->out_cnt_dev.reserve(nid * 4 + (size_t)B * 4))) return rc;
  int32_t* o_src = ctx->out_cnt_dev.as<int32_t>();
  int32_t* o_cnt = o_src + nid;
  if ((rc = sb_fuse_enqueue(ctx, method, rrf_k, w_dense, w_sparse, B, (const int64_t*)at(o_di), (const double*)at(o_ds),
                            (const int32_t*)at(o_dn), d_stride, (const int64_t*)at(o_si), (const double*)at(o_ss),
                            (const int32_t*)at(o_sn), s_stride, (const int64_t*)at(o_pi), (const double*)at(o_ps),
                            (const int32_t*)at(o_pn), p_stride, (const double*)at(o_ex), n_extra, e_stride, k,
                            ctx->out_ids_dev.as<int64_t>(), ctx->out_sc_dev.as<double>(), o_src, o_cnt, st)))
    return rc;
  if ((rc = ctx->pin_out.reserve(nid * 20 + (size_t)B * 4))) return rc;
  uint8_t* po = ctx->pin_out.as<uint8_t>();
  SB_CUDA(cudaMemcpyAsync(po, ctx->out_ids_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(po + nid * 8, ctx->out_sc_dev.p, nid * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaMemcpyAsync(po + nid * 16, o_src, nid * 4 + (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  memcpy(out_ids, po, nid * 8);
  memcpy(out_scores, po + nid * 8, nid * 8);
  memcpy(out_src, po + nid * 16, nid * 4);
  memcpy(out_counts, po + nid * 20, (size_t)B * 4);
  return SB_OK;
}

int sb_merge_shards_dev(sb_ctx* ctx, const int64_t* in_ids, const double* in_scores, const int32_t* in_counts,
                        int64_t shard_stride_bytes, int32_t G, int32_t B, int32_t k, int64_t* out_ids,
                        double* out_scores, int32_t* out_counts, void* stream) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_merge_shards_dev: ctx is NULL");
  SB_REQUIRE(G > 0 && B >= 0 && k > 0, SB_ERR_ARG, "sb_merge_shards_dev: bad G=%d B=%d k=%d", G, B, k);
  if (B == 0) return SB_OK;
  SB_REQUIRE(in_ids && in_scores && in_counts && out_ids && out_scores && out_counts, SB_ERR_ARG,
             "sb_merge_shards_dev: NULL buffer");
  int len = 1;
  while (len < G * k) len <<= 1;
  SB_REQUIRE((size_t)len * 16 <= ctx->smem_optin, SB_ERR_UNSUPPORTED, "sb_merge_shards_dev: G*k=%d too large", G * k);
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = pick_stream(ctx, stream);
  SB_CUDA(cudaFuncSetAttribute(merge_shards_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, len * 16));
  ctx->launches += 1;
  merge_shards_kernel<<<B, 256, (size_t)len * 16, st>>>(in_ids, in_scores, in_counts, shard_stride_bytes, G, B, k, len,
                                                        out_ids, out_scores, out_counts);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int sb_doc_chars_load(sb_ctx* ctx, const int32_t* n_chars, int64_t n_docs, int64_t id_base) {
  SB_REQUIRE(ctx != nullptr && n_docs >= 0 && (n_docs == 0 || n_chars), SB_ERR_ARG, "sb_doc_chars_load: bad arguments");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  SB_CUDA(cudaStreamSynchronize(ctx->stream));
  int rc = ctx->doc_chars_dev.reserve((size_t)std::max<int64_t>(n_docs, 1) * 4);
  if (rc) return rc;
  if (n_docs) SB_CUDA(cudaMemcpy(ctx->doc_chars_dev.p, n_chars, (size_t)n_docs * 4, cudaMemcpyHostToDevice));
  ctx->doc_chars_n = n_docs;
  ctx->doc_chars_base = id_base;
  return SB_OK;
}

int sb_select_dev(sb_ctx* ctx, const int64_t* cand_ids_dev, const void* cand_scores_dev, int32_t score_dtype,
                  const int32_t* cand_cnt_dev, int32_t B, int32_t k, int32_t top_k, int32_t max_tokens,
                  int64_t* out_ids_dev, void* out_scores_dev, int32_t* out_counts_dev, int32_t* out_tokens_dev,
                  void* stream) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_select_dev: ctx is NULL");
  SB_REQUIRE(B >= 0 && k > 0 && top_k > 0 && max_tokens >= 0, SB_ERR_ARG, "sb_select_dev: bad sizes");
  SB_REQUIRE(score_dtype == 0 || score_dtype == 1, SB_ERR_ARG, "sb_select_dev: score_dtype must be 0 (f32) or 1 (f64)");
  if (B == 0) return SB_OK;
  SB_REQUIRE(cand_ids_dev && cand_scores_dev && cand_cnt_dev && out_ids_dev && out_scores_dev && out_counts_dev &&
                 out_tokens_dev, SB_ERR_ARG, "sb_select_dev: NULL buffer");
  const size_t smem = (size_t)k * 12 + 16;
  SB_REQUIRE(smem <= 48 * 1024, SB_ERR_UNSUPPORTED, "sb_select_dev: k=%d too large", k);
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  SB_REQUIRE(ctx->doc_chars_dev.p != nullptr, SB_ERR_STATE, "sb_select_dev: no document lengths loaded (sb_doc_chars_load)");
  cudaStream_t st = pick_stream(ctx, stream);
  ctx->launches += 1;
  if (score_dtype == 0)
    select_docs_kernel<float><<<B, 128, smem, st>>>(cand_ids_dev, (const float*)cand_scores_dev, cand_cnt_dev, k, top_k,
                                                    max_tokens, ctx->doc_chars_dev.as<int32_t>(), ctx->doc_chars_n,
                                                    ctx->doc_chars_base, out_ids_dev, (float*)out_scores_dev,
                                                    out_counts_dev, out_tokens_dev);
  else
    select_docs_kernel<double><<<B, 128, smem, st>>>(cand_ids_dev, (const double*)cand_scores_dev, cand_cnt_dev, k, top_k,
                                                     max_tokens, ctx->doc_chars_dev.as<int32_t>(), ctx->doc_chars_n,
                                                     ctx->doc_chars_base, out_ids_dev, (double*)out_scores_dev,
                                                     out_counts_dev, out_tokens_dev);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

}  // extern "C"

int bm25_check_conditions(sb_ctx* ctx, const char* who, int B, const int32_t* f_off, const int32_t* f_field,
                          bool dense_too);   // bm25.cu

namespace {

// Host-buffer form of the whole path for one batch (single shard): pinned staging + ONE H2D of the queries / term ids
// (+ query word pieces), K1 + K2 + K3 (+ K5 rerank) enqueued on the context's stream through the device entry points, ONE
// D2H of the result lists.  What HybridRetriever.retrieve (hybrid.py:131-300) and rerank_node (nodes.py:138-227) do per
// query, for B queries per call, with no framework between the caller's buffers and the kernels.
struct RerankArgs {
  const int32_t* q_tok;   // [B, lq] host
  const int32_t* q_len;   // [B] host
  int32_t lq, S, k_out;
  int64_t* out_ids;       // [B, k_out]
  float* out_scores;      // [B, k_out]
  int32_t* out_counts;    // [B]
};

// Filtered (f_off != nullptr): one CSR of conditions per query, checked against both signals' columns before anything is
// enqueued and uploaded with the inputs; a batch without conditions takes the unfiltered calls.
int hybrid_host_call(sb_ctx* ctx, const char* who, const float* q, const int32_t* q_terms, const int32_t* q_off, int32_t B,
                     int32_t k, int32_t method, double rrf_k, double w_dense, double w_sparse, int64_t* out_ids,
                     double* out_scores, int32_t* out_src, int32_t* out_counts, const RerankArgs* rr,
                     const int32_t* f_off = nullptr, const int32_t* f_field = nullptr, const int32_t* f_code = nullptr) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "%s: ctx is NULL", who);
  SB_REQUIRE(B >= 0 && k > 0, SB_ERR_ARG, "%s: bad B=%d k=%d", who, B, k);
  if (B == 0) return SB_OK;
  SB_REQUIRE(q && q_off, SB_ERR_ARG, "%s: NULL input buffer", who);
  const int n_terms_q = q_off[B];
  SB_REQUIRE(n_terms_q >= 0 && (n_terms_q == 0 || q_terms), SB_ERR_ARG, "%s: bad query term buffers", who);
  int max_len = 0;
  for (int b = 0; b < B; ++b) {
    SB_REQUIRE(q_off[b + 1] >= q_off[b], SB_ERR_ARG, "%s: q_off must be non-decreasing", who);
    max_len = std::max(max_len, q_off[b + 1] - q_off[b]);
  }
  std::lock_guard<std::mutex> hl(ctx->hyb_mu);  // serialises whole calls: the staging buffers below belong to one call
  const int d = ctx->dense[0].d;
  SB_REQUIRE(ctx->dense[0].rows != nullptr && d > 0, SB_ERR_STATE, "%s: no dense index loaded in slot 0", who);
  const size_t qb = (size_t)B * d * 4, tb = (size_t)std::max(n_terms_q, 1) * 4, ob = (size_t)(B + 1) * 4;
  const size_t rb = rr ? (size_t)B * rr->lq * 4 + (size_t)B * 4 : 0;   // query word pieces + lengths
  const int n_conds = f_off ? f_off[B] : 0;
  const size_t cb = n_conds ? ob + (size_t)n_conds * 8 : 0;            // conditions: f_off | f_field | f_code
  const size_t in_bytes = qb + tb + ob + rb + cb;
  const size_t nid = (size_t)B * k;
  // device layout: inputs | dense ids sc cnt | sparse ids sc cnt | fused ids sc src cnt | reranked ids sc cnt
  const size_t cnt_b = ((size_t)B * 4 + 7) / 8 * 8;
  const size_t work_bytes = 2 * (nid * 16 + cnt_b);
  const size_t fused_bytes = (nid * 16 + nid * 4 + (size_t)B * 4 + 7) / 8 * 8;
  const size_t nrr = rr ? (size_t)B * rr->k_out : 0;
  const size_t rr_bytes = rr ? nrr * 12 + (size_t)B * 4 : 0;
  cudaStream_t st = ctx->stream;
  uint8_t *pi, *dv;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    int rc;
    if (f_off && (rc = bm25_check_conditions(ctx, who, B, f_off, f_field, true))) return rc;
    if ((rc = ctx->hyb_pin.reserve(std::max(in_bytes, std::max(fused_bytes, rr_bytes)) + 64))) return rc;
    if ((rc = ctx->hyb_dev.reserve((in_bytes + 7) / 8 * 8 + work_bytes + fused_bytes + rr_bytes + 64))) return rc;
    pi = ctx->hyb_pin.as<uint8_t>();
    dv = ctx->hyb_dev.as<uint8_t>();
    memcpy(pi, q, qb);
    if (n_terms_q) memcpy(pi + qb, q_terms, (size_t)n_terms_q * 4);
    memcpy(pi + qb + tb, q_off, ob);
    if (rr) {
      memcpy(pi + qb + tb + ob, rr->q_tok, (size_t)B * rr->lq * 4);
      memcpy(pi + qb + tb + ob + (size_t)B * rr->lq * 4, rr->q_len, (size_t)B * 4);
    }
    if (n_conds) {
      uint8_t* pc = pi + qb + tb + ob + rb;
      memcpy(pc, f_off, ob);
      memcpy(pc + ob, f_field, (size_t)n_conds * 4);
      memcpy(pc + ob + (size_t)n_conds * 4, f_code, (size_t)n_conds * 4);
    }
    SB_CUDA(cudaMemcpyAsync(dv, pi, in_bytes, cudaMemcpyHostToDevice, st));
  }
  const float* q_dev = reinterpret_cast<const float*>(dv);
  const int32_t* t_dev = reinterpret_cast<const int32_t*>(dv + qb);
  const int32_t* o_dev = reinterpret_cast<const int32_t*>(dv + qb + tb);
  const int32_t* qt_dev = reinterpret_cast<const int32_t*>(dv + qb + tb + ob);
  const int32_t* ql_dev = rr ? qt_dev + (size_t)B * rr->lq : nullptr;
  const int32_t* fo_dev = reinterpret_cast<const int32_t*>(dv + qb + tb + ob + rb);   // valid when n_conds > 0
  const int32_t* ff_dev = fo_dev + (B + 1);
  const int32_t* fc_dev = ff_dev + n_conds;
  uint8_t* w = dv + (in_bytes + 7) / 8 * 8;
  int64_t* d_ids = reinterpret_cast<int64_t*>(w);
  double* d_sc = reinterpret_cast<double*>(w + nid * 8);
  int32_t* d_cnt = reinterpret_cast<int32_t*>(w + nid * 16);
  uint8_t* w2 = w + nid * 16 + cnt_b;
  int64_t* s_ids = reinterpret_cast<int64_t*>(w2);
  double* s_sc = reinterpret_cast<double*>(w2 + nid * 8);
  int32_t* s_cnt = reinterpret_cast<int32_t*>(w2 + nid * 16);
  uint8_t* w3 = w2 + nid * 16 + cnt_b;
  int64_t* f_ids = reinterpret_cast<int64_t*>(w3);
  double* f_sc = reinterpret_cast<double*>(w3 + nid * 8);
  int32_t* f_src = reinterpret_cast<int32_t*>(w3 + nid * 16);
  int32_t* f_cnt = reinterpret_cast<int32_t*>(w3 + nid * 16 + nid * 4);
  uint8_t* w4 = w3 + fused_bytes;
  int64_t* r_ids = reinterpret_cast<int64_t*>(w4);
  float* r_sc = reinterpret_cast<float*>(w4 + nrr * 8);
  int32_t* r_cnt = reinterpret_cast<int32_t*>(w4 + nrr * 12);
  int rc;
  if (n_conds) {
    if ((rc = sb_dense_topk_filtered_dev(ctx, 0, q_dev, B, k, fo_dev, n_conds, ff_dev, fc_dev, d_ids, d_sc, d_cnt, st)))
      return rc;
    if ((rc = sb_bm25_topk_filtered_dev(ctx, t_dev, o_dev, B, n_terms_q, max_len, k, fo_dev, n_conds, ff_dev, fc_dev, s_ids,
                                        s_sc, s_cnt, st)))
      return rc;
  } else {
    if ((rc = sb_dense_topk_dev(ctx, 0, q_dev, B, k, d_ids, d_sc, d_cnt, st))) return rc;
    if ((rc = sb_bm25_topk_dev(ctx, t_dev, o_dev, B, n_terms_q, max_len, k, s_ids, s_sc, s_cnt, st))) return rc;
  }
  if ((rc = sb_fuse_dev(ctx, method, rrf_k, w_dense, w_sparse, B, d_ids, d_sc, d_cnt, k, s_ids, s_sc, s_cnt, k, nullptr,
                        nullptr, nullptr, 0, nullptr, 0, 0, k, f_ids, f_sc, f_src, f_cnt, st)))
    return rc;
  if (rr && (rc = sb_rerank_dev(ctx, qt_dev, ql_dev, rr->lq, f_ids, f_cnt, B, k, rr->S, rr->k_out, r_ids, r_sc, r_cnt, st)))
    return rc;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    if (rr)
      SB_CUDA(cudaMemcpyAsync(pi, w4, rr_bytes, cudaMemcpyDeviceToHost, st));
    else
      SB_CUDA(cudaMemcpyAsync(pi, w3, nid * 16 + nid * 4 + (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
  }
  if (rr) {
    memcpy(rr->out_ids, pi, nrr * 8);
    memcpy(rr->out_scores, pi + nrr * 8, nrr * 4);
    memcpy(rr->out_counts, pi + nrr * 12, (size_t)B * 4);
  } else {
    memcpy(out_ids, pi, nid * 8);
    memcpy(out_scores, pi + nid * 8, nid * 8);
    memcpy(out_src, pi + nid * 16, nid * 4);
    memcpy(out_counts, pi + nid * 16 + nid * 4, (size_t)B * 4);
  }
  return SB_OK;
}

}  // namespace

extern "C" {

int sb_hybrid_topk(sb_ctx* ctx, const float* q, const int32_t* q_terms, const int32_t* q_off, int32_t B, int32_t k,
                   int32_t method, double rrf_k, double w_dense, double w_sparse, int64_t* out_ids, double* out_scores,
                   int32_t* out_src, int32_t* out_counts) {
  SB_REQUIRE(B == 0 || (out_ids && out_scores && out_src && out_counts), SB_ERR_ARG, "sb_hybrid_topk: NULL output buffer");
  return hybrid_host_call(ctx, "sb_hybrid_topk", q, q_terms, q_off, B, k, method, rrf_k, w_dense, w_sparse, out_ids,
                          out_scores, out_src, out_counts, nullptr);
}

int sb_hybrid_topk_filtered(sb_ctx* ctx, const float* q, const int32_t* q_terms, const int32_t* q_off, int32_t B,
                            int32_t k, const int32_t* f_off, const int32_t* f_field, const int32_t* f_code,
                            int32_t method, double rrf_k, double w_dense, double w_sparse, int64_t* out_ids,
                            double* out_scores, int32_t* out_src, int32_t* out_counts) {
  SB_REQUIRE(B <= 0 || (out_ids && out_scores && out_src && out_counts), SB_ERR_ARG,
             "sb_hybrid_topk_filtered: NULL output buffer");
  SB_REQUIRE(B <= 0 || f_off != nullptr, SB_ERR_ARG, "sb_hybrid_topk_filtered: f_off is NULL");
  SB_REQUIRE(B <= 0 || f_off[B] == 0 || (f_field && f_code), SB_ERR_ARG, "sb_hybrid_topk_filtered: NULL conditions");
  return hybrid_host_call(ctx, "sb_hybrid_topk_filtered", q, q_terms, q_off, B, k, method, rrf_k, w_dense, w_sparse,
                          out_ids, out_scores, out_src, out_counts, nullptr, f_off, f_field, f_code);
}

int sb_hybrid_rerank_topk(sb_ctx* ctx, const float* q, const int32_t* q_terms, const int32_t* q_off, const int32_t* q_tok,
                          const int32_t* q_len, int32_t lq, int32_t B, int32_t k, int32_t k_out, int32_t S, int32_t method,
                          double rrf_k, double w_dense, double w_sparse, int64_t* out_ids, float* out_scores,
                          int32_t* out_counts) {
  SB_REQUIRE(B == 0 || (q_tok && q_len && out_ids && out_scores && out_counts), SB_ERR_ARG,
             "sb_hybrid_rerank_topk: NULL buffer");
  SB_REQUIRE(lq > 0 && k_out > 0 && S >= 8, SB_ERR_ARG, "sb_hybrid_rerank_topk: bad lq / k_out / S");
  RerankArgs rr{q_tok, q_len, lq, S, k_out, out_ids, out_scores, out_counts};
  return hybrid_host_call(ctx, "sb_hybrid_rerank_topk", q, q_terms, q_off, B, k, method, rrf_k, w_dense, w_sparse, nullptr,
                          nullptr, nullptr, nullptr, &rr);
}

}  // extern "C"
