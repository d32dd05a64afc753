// common.cuh -- shared host/device helpers for libsentio_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/sentio_b200.h"

// ------------------------------------------------------------------ error plumbing
void sb_set_error(const char* fmt, ...);

#define SB_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      sb_set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__,    \
                   cudaGetErrorString(_e));                                                   \
      return SB_ERR_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

#define SB_REQUIRE(cond, code, ...)  \
  do {                               \
    if (!(cond)) {                   \
      sb_set_error(__VA_ARGS__);     \
      return (code);                 \
    }                                \
  } while (0)

// ------------------------------------------------------------------ device buffers (grow-only scratch)
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return SB_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + (bytes >> 2) + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
      sb_set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
      return SB_ERR_CUDA;
    }
    cap = want;
    return SB_OK;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

struct PinBuf {
  void* p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return SB_OK;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + (bytes >> 2) + 256;
    cudaError_t e = cudaMallocHost(&p, want);
    if (e != cudaSuccess) {
      sb_set_error("cudaMallocHost(%zu) failed: %s", want, cudaGetErrorString(e));
      return SB_ERR_CUDA;
    }
    cap = want;
    return SB_OK;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

// ------------------------------------------------------------------ index state
struct DenseIndex {
  int64_t n = 0;        // valid rows
  int64_t n_pad = 0;    // rows the scans cover: round_up(n, 128)
  int64_t n_cap = 0;    // rows allocated in rows / inv_norm / every tag column (>= n_pad, multiple of 128); rows in
                        // [n, n_cap) are zero with inv_norm 0 and tag code -1
  int32_t d = 0;        // logical dimension
  int32_t d_pad = 0;    // stored row length in halves (multiple of 8 -> 16 B aligned rows)
  int64_t id_base = 0;
  int32_t metric = SB_METRIC_COSINE;
  __half* rows = nullptr;    // [n_cap][d_pad] y = fp16(x / ||x||) (Cosine: also fp16 input verbatim)
  // per-row scan scale, what the scans multiply their fp32 dot product by: Cosine 1/||y|| of the STORED fp16 row (0 for
  // zero rows); Dot / Euclid (float)c
  float* inv_norm = nullptr; // [n_cap]
  // Dot / Euclid (DESIGN.md K1e): the stored vector is v = c * y with c = ||x|| / ||y|| (fp64, 0 for zero rows)
  double* cfac = nullptr;    // [n_cap], nullptr for Cosine
  float* hh = nullptr;       // [n_cap] Euclid only: h >= ||v||^2 / 2 rounded up to fp32
  double rho_max = 0.0;      // >= max ||v|| over every row ever stored since the load (an upsert may raise it)
  double h_max = 0.0;        // Euclid: >= max h, likewise
  // float32 storage (DESIGN.md K1g): the caller's rows x next to everything above, which the scans still read.  The exact
  // stage scores x; sigma_max >= max over rows ever stored of ||y^ - x^|| (Cosine) or ||c y - x|| (Dot / Euclid)
  int32_t storage = SB_STORAGE_F16;
  float* rows32 = nullptr;   // [n_cap][d_pad] fp32, zero padded; nullptr for float16 storage
  double sigma_max = 0.0;
  // uint8 storage (DESIGN.md K1i): the caller's integer rows x, one byte per dimension, INSTEAD of `rows` (which stays
  // nullptr); d_pad = round_up(d, 64).  inv_norm is the scan scale (Cosine fl32(1/||x||), Dot / Euclid 1), hh = ||x||^2 / 2
  // rounded up (Euclid), cfac is not allocated and sigma_max stays 0: the scan reads the vector it scores.
  uint8_t* rows8 = nullptr;  // [n_cap][d_pad]
  // cached CUtensorMap (128 bytes, 64-byte aligned) over rows[0, n_pad) (uint8: rows8) for the wgmma batched scan;
  // valid iff tm_rows_ptr == rows (rows8) and tm_n_pad == n_pad (an append within capacity keeps `rows` but widens n_pad)
  alignas(64) unsigned char tm_rows[128] = {0};
  const void* tm_rows_ptr = nullptr;
  int64_t tm_n_pad = 0;
  // payload index for filtered search (sb_dense_tags_load): tags[f][row] = dictionary code of field f, -1 = key absent;
  // nullptr = field f not loaded.  Dropped by sb_dense_load.
  int32_t* tags[SB_MAX_TAG_FIELDS] = {};
  // numeric payload columns for range filters (sb_dense_values_load): vals[f][row] = the fp64 value, NaN = none;
  // nullptr = not loaded.  Same capacity and mutation rules as the tag columns.  Dropped by sb_dense_load.
  double* vals[SB_MAX_VALUE_FIELDS] = {};
};

struct Bm25Index {
  int64_t n_docs = 0, n_terms = 0, nnz = 0;
  int64_t id_base = 0;
  int32_t variant = 0;
  double k1 = 1.5, b = 0.75, delta = 1.0, avgdl = 0.0;
  int64_t* indptr = nullptr;   // [V+1]
  int32_t* post_doc = nullptr; // [nnz]
  double* post_ratio = nullptr; // [nnz] query-independent tf*(k1+1)/(tf+dnorm[doc]) (fp64, exact op order)
  double* dnorm = nullptr;     // [n_docs]  k1*(1-b+b*dl/avgdl), same op order as rank_bm25
  double* idf = nullptr;       // [V]
  // head terms (df >= n_docs / 4) additionally keep a DENSE ratio row: dense_ratio[slot][doc] (0.0 where the doc has no
  // posting); dense_of_term[t] = slot or -1.  The scoring kernel streams these rows with fully predictable addresses
  int32_t n_dense = 0;
  int32_t* dense_of_term = nullptr;  // [V]
  double* dense_ratio = nullptr;     // [n_dense][n_docs]
  // payload index for filtered BM25 (sb_bm25_tags_load): tags[f][doc] = dictionary code of field f, -1 = key absent;
  // nullptr = field f not loaded.  They belong to the installed index: installing another one frees them
  int32_t* tags[SB_MAX_TAG_FIELDS] = {};
};

struct CeModel;      // cross_encoder.cu
struct CeDocTokens;  // cross_encoder.cu
struct Bm25Build;    // bm25_build.cu

struct sb_ctx {
  int device = 0;
  int num_sms = 0;
  size_t smem_optin = 0;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  DenseIndex dense[SB_MAX_DENSE_SLOTS];
  Bm25Index bm25;
  CeModel* ce = nullptr;   // reranker (sb_ce_load)
  CeModel* enc = nullptr;  // query / document embedder (sb_enc_load)
  CeDocTokens* ce_tokens = nullptr;
  Bm25Build* bm25_build = nullptr;  // GPU index build in progress (sb_bm25_build_tokens .. sb_bm25_build_finish)
  int dense_mode = 0;  // 0 = auto, 1 = CUDA-core scan only, 2 = wgmma batched scan whenever eligible
  int dense_sample_per_cta = 2;  // tiles per CTA of the sampling pass (env SB_DENSE_SAMPLE)
  int dense_prefetch = 0;      // boxes prefetched into L2 beyond the ring (env SB_DENSE_PREFETCH; 0 = off)
  int dense_max_stages = 8;    // cap on the TMA ring depth (env SB_DENSE_STAGES)
  // bookkeeping: kernels launched by this library, optional per-kernel CUDA-event timing (bench.py roofline leg)
  uint64_t launches = 0;
  bool prof_on = false;
  struct ProfRec { int id; cudaEvent_t a, b; };
  std::vector<ProfRec> prof_recs;
  std::vector<cudaEvent_t> prof_pool;
  // scratch
  DevBuf q_dev, cand_dev, out_ids_dev, out_sc_dev, out_cnt_dev, misc_dev, misc2_dev, misc3_dev, acc_dev;
  DevBuf qn_dev;     // dense: normalised fp32 queries [B][d_pad] fed to the scans
  DevBuf reco_dev;   // dense recommendation (DESIGN.md K1j): operand rows, per-example bounds, keys and intervals
  DevBuf qaux_dev;   // dense: per-query eps [B] fp32 | fallback flags [B] i32
  DevBuf fb_count_dev;   // dense: [1] u64, queries answered by the exact fallback kernel (sb_dense_fallback_count)
  DevBuf sigma_dev;      // dense float32 storage: [1] u64, bits of the largest sigma of the rows one load / upsert stores
  DevBuf filt_dev;       // filtered dense: per-query counts / state | one chunk's filter programs | match mask
  PinBuf filt_pin;       // filtered dense: host copies of the per-query counts / state and the programs
  // grouped dense search (sb_dense_groups): result [B][L][G] | one round's prefixes | replicated queries | completions
  DevBuf grp_res_dev, grp_round_dev, grp_q_dev, grp_cmp_dev;
  std::vector<int64_t> grp_rounds;   // [r]: grouped queries answered in r + 1 rounds (sb_dense_group_rounds)
  DevBuf doc_chars_dev;  // K7: characters of every document's usable text (0 = blank), sb_doc_chars_load
  int64_t doc_chars_n = 0, doc_chars_base = 0;
  PinBuf pin_in, pin_out;
  // sb_hybrid_topk: staging of one whole-path call (its own buffers and lock: the inner entry points take `mu`)
  std::mutex hyb_mu;
  PinBuf hyb_pin;
  DevBuf hyb_dev;
};

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    int cur = -1;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

// kernel ids for sb_profile_read
enum { SB_PROF_DENSE_SCAN = 0, SB_PROF_DENSE_MERGE = 1, SB_PROF_BM25_SCORE = 2, SB_PROF_BM25_SELECT = 3,
       SB_PROF_FUSE = 4, SB_PROF_CE = 5, SB_PROF_DENSE_SAMPLE = 6, SB_PROF_DENSE_FILTER = 7,
       SB_PROF_DENSE_GATHER = 8, SB_PROF_DENSE_GROUP_COLLECT = 9, SB_PROF_DENSE_GROUP_ASSEMBLE = 10,
       SB_PROF_COUNT = 11 };

static inline cudaEvent_t prof_event(sb_ctx* ctx) {
  if (!ctx->prof_pool.empty()) {
    cudaEvent_t e = ctx->prof_pool.back();
    ctx->prof_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}
// bracket `n_kernels` launches of kernel `id` on stream st with an event pair when profiling is enabled
struct ProfScope {
  sb_ctx* ctx;
  cudaStream_t st;
  cudaEvent_t b = nullptr;
  ProfScope(sb_ctx* c, int id, cudaStream_t s, int n_kernels = 1) : ctx(c), st(s) {
    ctx->launches += (uint64_t)n_kernels;
    if (ctx->prof_on) {
      cudaEvent_t a = prof_event(ctx);
      b = prof_event(ctx);
      cudaEventRecord(a, st);
      ctx->prof_recs.push_back({id, a, b});
    }
  }
  ~ProfScope() {
    if (b) cudaEventRecord(b, st);
  }
};

// true when [p, p + bytes) is page-locked host memory the copy engines can reach directly (cudaMallocHost / registered)
static inline bool host_ptr_is_pinned(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeHost;
}

static inline cudaStream_t pick_stream(sb_ctx* ctx, void* stream) {
  return stream ? reinterpret_cast<cudaStream_t>(stream) : ctx->stream;
}

// ------------------------------------------------------------------ device helpers
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t f32_orderable(float f) {
  uint32_t u = __float_as_uint(f);
  return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float orderable_f32(uint32_t u) {
  u ^= (u >> 31) ? 0x80000000u : 0xffffffffu;
  return __uint_as_float(u);
}
__device__ __forceinline__ uint64_t f64_orderable(double d) {
  uint64_t u = (uint64_t)__double_as_longlong(d);
  return u ^ ((u >> 63) ? 0xffffffffffffffffull : 0x8000000000000000ull);
}
__device__ __forceinline__ double orderable_f64(uint64_t u) {
  u ^= (u >> 63) ? 0x8000000000000000ull : 0xffffffffffffffffull;
  return __longlong_as_double((long long)u);
}
// composite key: larger = better.  hi 32 = orderable score, lo 32 = ~idx (lower idx wins ties).
__device__ __forceinline__ uint64_t make_key32(float score, uint32_t idx) {
  return ((uint64_t)f32_orderable(score) << 32) | (uint64_t)(~idx);
}
__device__ __forceinline__ uint32_t key32_idx(uint64_t k) { return ~(uint32_t)(k & 0xffffffffu); }
__device__ __forceinline__ float key32_score(uint64_t k) { return orderable_f32((uint32_t)(k >> 32)); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}


// Radix-select helper, called by ONE full warp: scan the 256-bin histogram from the top (DESC) or the bottom and find the
// bin where the running count first reaches `need`.  out[0] = bin, out[1] = rank inside the bin (need - count of the bins
// before it), out[2] = the bin's count.  Lane l owns 8 consecutive bins in scan order; one shuffle scan across lanes.
template <bool DESC>
__device__ __forceinline__ void warp_select_bin(const int* hist, int need, int lane, int* out) {
  int c[8];
  int s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int b = DESC ? 255 - 8 * lane - i : 8 * lane + i;
    c[i] = hist[b];
    s += c[i];
  }
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  const int excl = incl - s;
  const bool mine = excl < need && need <= incl;
  const unsigned m = __ballot_sync(0xffffffffu, mine);
  if (mine) {
    int cum = excl;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (cum + c[i] >= need) {
        out[0] = DESC ? 255 - 8 * lane - i : 8 * lane + i;
        out[1] = need - cum;
        out[2] = c[i];
        break;
      }
      cum += c[i];
    }
  }
  if (m == 0u && lane == 31) {  // fewer than `need` keys in total (callers avoid it): same answer as a full serial scan
    out[0] = DESC ? 0 : 255;
    out[1] = need - incl;
    out[2] = hist[DESC ? 0 : 255];
  }
}

// ---- mbarrier / bulk-copy (TMA engine, SASS UBLKCP) wrappers
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// 1-D bulk async copy global -> shared, completion signalled on an mbarrier (bytes % 16 == 0, 16 B aligned).
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// barrier + OR reduction of a predicate over the participating threads
__device__ __forceinline__ bool named_bar_or(int id, int nthreads, bool pred) {
  uint32_t r;
  asm volatile(
      "{\n"
      ".reg .pred p, q;\n"
      "setp.ne.u32 p, %3, 0;\n"
      "bar.red.or.pred q, %1, %2, p;\n"
      "selp.u32 %0, 1, 0, q;\n"
      "}\n"
      : "=r"(r)
      : "r"(id), "r"(nthreads), "r"((uint32_t)pred)
      : "memory");
  return r != 0;
}

#endif  // __CUDACC__
