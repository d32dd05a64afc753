// dense_mma.cuh -- interface of the wgmma batched-query dense scan (dense_mma.cu) and the pieces it shares with dense.cu.
#pragma once
#include "common.cuh"

// Filtered search (DESIGN.md K1c): the match mask of one chunk of queries and what the host learned from it.  A scan
// given a DenseFilter appends only rows whose mask bit is set and leaves queries with state 1 (answered by the gather
// path) alone.
struct DenseFilter {
  const uint32_t* mask;        // [n_pad / 32][qs] match bits; column = query index inside the chunk
  int32_t qs;
  const int32_t* state;        // device [nq]: 1 = answered by the gather path
  const int32_t* state_host;   // host copy of state
  int64_t c_min;               // fewest matching rows among the scanned queries (sizes the wgmma scan)
};

// true when the batched tensor-core scan can serve this index / batch (B >= 16, d_pad % 64 == 0, corpus >= 8192 rows)
bool dense_mma_eligible(const sb_ctx* ctx, const DenseIndex& ix, int B);

// q_pad: [B][d_pad] fp32 device (zero padded).  Enqueues sampling passes + full passes + the exact stage for groups of
// <= 256 queries (one HBM pass over the corpus per group).
int dense_mma_topk_enqueue(sb_ctx* ctx, DenseIndex& ix, const float* q_pad, int B, int k, int64_t* out_ids,
                           double* out_scores, int32_t* out_counts, cudaStream_t st, const DenseFilter* flt = nullptr);

// dense.cu: normalised fp32 queries / fp16 operand rows / eps / cleared fallback flags for `rows` >= B operand rows, and
// for a Euclid slot the fp32 query norms r (*rq_out; nullptr for Cosine / Dot).  Flags of Dot / Euclid queries whose
// keys the scans cannot bound are raised here already (DESIGN.md K1e).
int dense_prep_queries(sb_ctx* ctx, const DenseIndex& ix, const float* q_pad, int B, int rows, bool mma, float** qn_out,
                       __half* q16, float** eps_out, int32_t** fb_out, float** rq_out, cudaStream_t st);
// Recommendation (DESIGN.md K1j): request r owns examples [ex0, ex0 + m) of the padded example rows, the first n_pos
// positive, merged by strategy (SB_RECO_*).
struct RecoReq {
  int32_t ex0, m, n_pos, strategy;
};
// R validated requests over M examples (ex_pad: [M][d_pad] fp32 device), programs as sb_dense_topk_where (host arrays;
// p_off == nullptr: unfiltered), k <= 1024, a Cosine or Dot slot with rows: the exact top-k of every request.
int dense_reco_enqueue(sb_ctx* ctx, DenseIndex& ix, const float* ex_pad, int M, const RecoReq* req, int R, int k,
                       const int32_t* p_off, const sb_pred* prog, const int32_t* pool, int64_t* out_ids,
                       double* out_scores, int32_t* out_counts, cudaStream_t st);
// dense.cu: the match mask of queries [c0, c0 + nq) (nq <= 256) of validated programs; bit (row % 32) of
// (*mask)[(row / 32) * *qs + q - c0].  The mask lives in the context's filter buffer until the next filtered call.
int dense_where_mask(sb_ctx* ctx, DenseIndex& ix, const int32_t* p_off, const sb_pred* prog, const int32_t* pool, int c0,
                     int nq, const uint32_t** mask, int* qs, cudaStream_t st);
// dense.cu: brute-force fp64 answer for every query whose fallback flag is raised (one CTA per query, idle CTAs exit)
int dense_fallback_enqueue(sb_ctx* ctx, const DenseIndex& ix, const float* q_pad, int B, int k, const int32_t* fb,
                           int64_t* out_ids, double* out_scores, int32_t* out_counts, cudaStream_t st,
                           const DenseFilter* flt = nullptr);
