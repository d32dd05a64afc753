// mmr.cu -- K4: semantic-similarity and greedy-MMR scorer signals over the fused candidate set.
//
// Replaces SemanticSimilarityScorer.score / MMRScorer.score (reference src/core/retrievers/scorers.py:152-191,222-273),
// i.e. an O(n^3) Python loop of np.dot / np.linalg.norm calls, by: gather candidate vectors -> fp64 cosine to the
// query -> fp64 cosine Gram matrix -> single-CTA greedy selection with an incrementally maintained max-redundancy.
// Latency bound (n <= a few hundred candidates); all arithmetic fp64 like the NumPy reference.
#include <algorithm>
#include <string.h>

#include "common.cuh"

namespace {

constexpr int kGreedyThreads = 1024;

// candidates by id from the stored corpus -> fp32 matrix: the fp16 rows, or a float32 / uint8 slot's x (what its search
// scores)
template <typename T>
__global__ void mmr_gather_kernel(const T* rows, int d, int d_pad, int64_t n_rows, int64_t id_base,
                                  const int64_t* ids, int n, float* out) {
  const int r = blockIdx.x;
  if (r >= n) return;
  const int64_t idx = ids[r] - id_base;
  const bool ok = idx >= 0 && idx < n_rows;
  for (int i = threadIdx.x; i < d; i += blockDim.x)
    out[(size_t)r * d + i] = ok ? (float)rows[(size_t)idx * d_pad + i] : 0.f;
}

// one warp per candidate: dot(q, c_i), |c_i|^2 ; warp 0 of block 0 also |q|^2
__global__ void mmr_rel_kernel(const float* __restrict__ q, const float* __restrict__ C, int n, int d,
                               double* __restrict__ dotq, double* __restrict__ nrm2, double* __restrict__ qq) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w == 0) {
    double s = 0.0;
    for (int i = lane; i < d; i += 32) s += (double)q[i] * (double)q[i];
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) qq[0] = s;
  }
  if (w >= n) return;
  const float* c = C + (size_t)w * d;
  double dq = 0.0, cc = 0.0;
  for (int i = lane; i < d; i += 32) {
    const double x = (double)c[i];
    dq += x * (double)q[i];
    cc += x * x;
  }
  for (int o = 16; o; o >>= 1) {
    dq += __shfl_xor_sync(0xffffffffu, dq, o);
    cc += __shfl_xor_sync(0xffffffffu, cc, o);
  }
  if (lane == 0) {
    dotq[w] = dq;
    nrm2[w] = cc;
  }
}

// cosine Gram matrix, one warp per (i, j >= i) pair; sim[i][j] = sim[j][i] = dot / (|c_i| * |c_j|) (0 if denom == 0)
__global__ void mmr_gram_kernel(const float* __restrict__ C, int n, int d, const double* __restrict__ nrm2,
                                double* __restrict__ sim) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (int64_t)n * n) return;
  const int i = (int)(w / n), j = (int)(w % n);
  if (j < i) return;
  const float* a = C + (size_t)i * d;
  const float* b = C + (size_t)j * d;
  double s = 0.0;
  for (int t = lane; t < d; t += 32) s += (double)a[t] * (double)b[t];
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const double den = sqrt(nrm2[i]) * sqrt(nrm2[j]);
    const double v = den != 0.0 ? s / den : 0.0;
    sim[(size_t)i * n + j] = v;
    sim[(size_t)j * n + i] = v;
  }
}

struct GreedyParams {
  int n;
  const double* dotq;
  const double* nrm2;
  const double* qq;
  const double* sim;  // may be NULL when out_mmr is NULL
  double w_sem, lambda, w_mmr;
  double* out_sem;  // may be NULL
  double* out_mmr;  // may be NULL
  double* rel_scratch;  // [n]
  double* red_scratch;  // [n]
};

__global__ void __launch_bounds__(kGreedyThreads, 1) mmr_greedy_kernel(const GreedyParams p) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = p.n;
  __shared__ double s_best[32];
  __shared__ int s_bidx[32];
  __shared__ double s_pick_score;
  __shared__ int s_pick;
  const double qn = sqrt(p.qq[0]);
  double* rel = p.rel_scratch;
  double* red = p.red_scratch;
  for (int i = tid; i < n; i += kGreedyThreads) {
    const double dn = sqrt(p.nrm2[i]);
    const double den = qn * dn;
    const double r = den != 0.0 ? p.dotq[i] / den : 0.0;
    rel[i] = r;
    red[i] = 0.0;
    if (p.out_sem) p.out_sem[i] = (qn > 0.0 && dn > 0.0) ? __dmul_rn(r, p.w_sem) : 0.0;
    if (p.out_mmr) p.out_mmr[i] = 0.0;
  }
  if (!p.out_mmr) return;
  __syncthreads();
  const double oml = 1.0 - p.lambda;
  // selected flag is encoded by red[i] = NaN-free sentinel: keep a bitmask in registers per owned candidate
  // (each thread owns candidates tid, tid + 1024, ... ; n <= 4096 -> at most 4)
  unsigned sel_mask = 0;
  for (int it = 0; it < n; ++it) {
    double best = -1.0;
    int bidx = -1;
    int slot = 0;
    for (int i = tid; i < n; i += kGreedyThreads, ++slot) {
      if (sel_mask & (1u << slot)) continue;
      const double sc = __dsub_rn(__dmul_rn(p.lambda, rel[i]), __dmul_rn(oml, red[i]));
      if (sc > best) {  // strict: the first (lowest) index wins ties inside one thread
        best = sc;
        bidx = i;
      }
    }
    // warp argmax by (score desc, idx asc); bidx == -1 means "nothing > -1.0"
    for (int o = 16; o; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      const bool take = (oi >= 0) && (bidx < 0 || ob > best || (ob == best && oi < bidx));
      if (take) {
        best = ob;
        bidx = oi;
      }
    }
    if (lane == 0) {
      s_best[warp] = best;
      s_bidx[warp] = bidx;
    }
    __syncthreads();
    if (warp == 0) {
      best = s_best[lane];
      bidx = s_bidx[lane];
      for (int o = 16; o; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
        const bool take = (oi >= 0) && (bidx < 0 || ob > best || (ob == best && oi < bidx));
        if (take) {
          best = ob;
          bidx = oi;
        }
      }
      if (lane == 0) {
        s_pick = bidx;
        s_pick_score = best;
      }
    }
    __syncthreads();
    const int pick = s_pick;
    if (pick < 0) break;  // reference: best_idx is None -> break
    const double pscore = s_pick_score;
    slot = 0;
    for (int i = tid; i < n; i += kGreedyThreads, ++slot) {
      if (i == pick) {
        sel_mask |= (1u << slot);
        p.out_mmr[i] = __dmul_rn(pscore, p.w_mmr);
      } else if (!(sel_mask & (1u << slot))) {
        const double s = p.sim[(size_t)i * n + pick];
        if (s > red[i]) red[i] = s;
      }
    }
    __syncthreads();
  }
  __syncthreads();
  for (int i = tid; i < n; i += kGreedyThreads) {
    double m = p.out_mmr[i];
    if (m == 0.0) m = __dmul_rn(__dmul_rn(rel[i], p.w_mmr), p.lambda);
    p.out_mmr[i] = m > 0.0 ? m : 0.0;  // max(0.0, m)
  }
}

}  // namespace

extern "C" {

int sb_semantic_mmr(sb_ctx* ctx, int slot, const float* q, int32_t d, const float* cand, const int64_t* cand_ids,
                    int32_t n, double w_sem, double lambda, double w_mmr, double* out_sem, double* out_mmr) {
  SB_REQUIRE(ctx != nullptr, SB_ERR_ARG, "sb_semantic_mmr: ctx is NULL");
  SB_REQUIRE(n >= 0 && d > 0 && q, SB_ERR_ARG, "sb_semantic_mmr: bad arguments");
  if (n == 0) return SB_OK;
  SB_REQUIRE(n <= 4096, SB_ERR_UNSUPPORTED, "sb_semantic_mmr: at most 4096 candidates (got %d)", n);
  SB_REQUIRE(cand || cand_ids, SB_ERR_ARG, "sb_semantic_mmr: neither candidate vectors nor ids given");
  SB_REQUIRE(out_sem || out_mmr, SB_ERR_ARG, "sb_semantic_mmr: no output requested");
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  cudaStream_t st = ctx->stream;
  int rc;
  // device layout: [q d f32][C n*d f32] | doubles: dotq[n] nrm2[n] qq[2] rel[n] red[n] sem[n] mmr[n] sim[n*n]
  const size_t fbytes = ((size_t)d + (size_t)n * d) * 4;
  const size_t nd = (size_t)n;
  const size_t dcount = 6 * nd + 2 + (out_mmr ? nd * nd : 0);
  if ((rc = ctx->misc_dev.reserve(fbytes + 64))) return rc;
  if ((rc = ctx->misc2_dev.reserve(dcount * 8 + 64))) return rc;
  float* qd = ctx->misc_dev.as<float>();
  float* Cd = qd + d;
  double* dotq = ctx->misc2_dev.as<double>();
  double* nrm2 = dotq + nd;
  double* qq = nrm2 + nd;
  double* rel = qq + 2;
  double* red = rel + nd;
  double* sem = red + nd;
  double* mmr = sem + nd;
  double* sim = mmr + nd;
  SB_CUDA(cudaMemcpyAsync(qd, q, (size_t)d * 4, cudaMemcpyHostToDevice, st));
  if (cand) {
    SB_CUDA(cudaMemcpyAsync(Cd, cand, (size_t)n * d * 4, cudaMemcpyHostToDevice, st));
  } else {
    SB_REQUIRE(slot >= 0 && slot < SB_MAX_DENSE_SLOTS, SB_ERR_ARG, "sb_semantic_mmr: bad slot %d", slot);
    const DenseIndex& ix = ctx->dense[slot];
    SB_REQUIRE(ix.n > 0 && ix.d == d, SB_ERR_STATE,
               "sb_semantic_mmr: dense slot %d is empty or has dimension %d != %d", slot, ix.d, d);
    if ((rc = ctx->misc3_dev.reserve(nd * 8))) return rc;
    SB_CUDA(cudaMemcpyAsync(ctx->misc3_dev.p, cand_ids, nd * 8, cudaMemcpyHostToDevice, st));
    if (ix.storage == SB_STORAGE_U8)
      mmr_gather_kernel<uint8_t><<<n, 128, 0, st>>>(ix.rows8, ix.d, ix.d_pad, ix.n, ix.id_base,
                                                    ctx->misc3_dev.as<int64_t>(), n, Cd);
    else if (ix.storage == SB_STORAGE_F32)
      mmr_gather_kernel<float><<<n, 128, 0, st>>>(ix.rows32, ix.d, ix.d_pad, ix.n, ix.id_base,
                                                  ctx->misc3_dev.as<int64_t>(), n, Cd);
    else
      mmr_gather_kernel<__half><<<n, 128, 0, st>>>(ix.rows, ix.d, ix.d_pad, ix.n, ix.id_base,
                                                   ctx->misc3_dev.as<int64_t>(), n, Cd);
    SB_CUDA(cudaGetLastError());
  }
  {
    const int warps = n + 1;
    const int blocks = (warps * 32 + 255) / 256;
    mmr_rel_kernel<<<blocks, 256, 0, st>>>(qd, Cd, n, d, dotq, nrm2, qq);
    SB_CUDA(cudaGetLastError());
  }
  if (out_mmr) {
    const int64_t warps = (int64_t)n * n;
    const unsigned blocks = (unsigned)((warps * 32 + 255) / 256);
    mmr_gram_kernel<<<blocks, 256, 0, st>>>(Cd, n, d, nrm2, sim);
    SB_CUDA(cudaGetLastError());
  }
  GreedyParams gp;
  gp.n = n;
  gp.dotq = dotq;
  gp.nrm2 = nrm2;
  gp.qq = qq;
  gp.sim = out_mmr ? sim : nullptr;
  gp.w_sem = w_sem;
  gp.lambda = lambda;
  gp.w_mmr = w_mmr;
  gp.out_sem = out_sem ? sem : nullptr;
  gp.out_mmr = out_mmr ? mmr : nullptr;
  gp.rel_scratch = rel;
  gp.red_scratch = red;
  mmr_greedy_kernel<<<1, kGreedyThreads, 0, st>>>(gp);
  SB_CUDA(cudaGetLastError());
  if (out_sem) SB_CUDA(cudaMemcpyAsync(out_sem, sem, nd * 8, cudaMemcpyDeviceToHost, st));
  if (out_mmr) SB_CUDA(cudaMemcpyAsync(out_mmr, mmr, nd * 8, cudaMemcpyDeviceToHost, st));
  SB_CUDA(cudaStreamSynchronize(st));
  return SB_OK;
}

}  // extern "C"
