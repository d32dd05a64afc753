"""HybridPipeline -- batched, optionally sharded, arrays-in / arrays-out form of the hot path.

One process per GPU.  Each rank owns a contiguous doc-id range of the corpus (dense rows + BM25 postings with
corpus-global idf/avgdl).  A batch of B queries runs:

    local K1 dense top-k  +  local K2 BM25 top-k          (raw scores, shard-local)
    ONE all-gather of the per-rank record {dense ids/scores/counts, sparse ids/scores/counts}   (world > 1)
    K6 merge to the GLOBAL top-k per signal  ->  K3 fusion on global ranks  ->  [K5 rerank]

``*_dev`` methods keep everything on the device on torch's current stream (bench.py's resident leg);
``search_*`` methods take host NumPy inputs and return host NumPy outputs (the e2e leg).
torch / torch.distributed are plumbing only (device buffers, streams, the NCCL all-gather).
"""
from __future__ import annotations

from typing import Sequence

import numpy as np

from .engine import B200Engine
from .index import Bm25IndexData


def plan_layout(world: int, index_gb: float, mode: str = "auto", corpus_shards: int = 0, budget_gb: float = 64.0):
    """Multi-GPU layout = C corpus shards x world / C query groups -> (C, n_groups).

    ``corpus``: C = world (every rank holds 1/world of the corpus; one all-gather per batch); ``queries``: C = 1
    (replicated corpus, no collective); ``auto``: the smallest divisor C of ``world`` whose shard (index_gb / C) fits
    ``budget_gb`` -- partition only as much as capacity requires; an explicit ``corpus_shards`` overrides ``mode``."""
    if world < 1:
        raise ValueError("world must be >= 1")
    if corpus_shards:
        C = int(corpus_shards)
    elif mode == "corpus":
        C = world
    elif mode == "queries":
        C = 1
    elif mode == "auto":
        C = next(c for c in range(1, world + 1) if world % c == 0 and (index_gb / c <= budget_gb or c == world))
    else:
        raise ValueError(f"unknown layout mode {mode!r}")
    if C < 1 or world % C:
        raise ValueError(f"corpus_shards={C} must divide world={world}")
    return C, world // C


class HybridPipeline:
    def __init__(self, device: int | None = 0, rank: int = 0, world: int = 1, group=None, engine=None):
        """``engine`` may be injected (the CPU/gloo tests pass an oracle-backed double together with device=None);
        the product path always builds a real ``B200Engine`` on ``cuda:device``."""
        import torch

        self.torch = torch
        self.device = device
        self.rank, self.world, self.group = rank, world, group
        if engine is None:
            if device is None:
                raise ValueError("HybridPipeline needs a CUDA device (there is no CPU path)")
            torch.cuda.set_device(device)
            engine = B200Engine(device)
        self.engine = engine
        self._torch_device = "cpu" if device is None else f"cuda:{device}"
        self.id_base = 0
        self._bufs = {}
        # optional per-stage CUDA-event timing of the sharded path (bench.py's `partitioned` leg)
        self.stage_timing = False
        self._stage_events: list = []
        self.stage_counts: dict = {}

    # ------------------------------------------------------------------ loading
    def load_dense(self, vecs: np.ndarray, id_base: int = 0) -> None:
        self.engine.load_dense(vecs, id_base=id_base, slot=0)
        self.id_base = id_base

    def load_bm25(self, data: Bm25IndexData, id_base: int = 0) -> None:
        self.engine.load_bm25(data, id_base=id_base)

    def build_bm25_sharded(self, flat_tokens: np.ndarray, doc_offsets: np.ndarray, id_base: int = 0, variant: str = "okapi",
                           k1: float = 1.5, b: float = 0.75, epsilon: float = 0.25, delta: float = 1.0,
                           export: bool = False) -> Bm25IndexData:
        """Index build of a PARTITIONED corpus without a host-side global index: every rank builds the postings of its own
        doc range on its GPU (sb_bm25_build_*), the per-shard (term, df, doc / token counts) are all-gathered -- a few
        hundred KB -- and every rank derives the same corpus-global idf / avgdl (index.global_bm25_stats: bit-identical to
        the single-index build), which its shard is then scored with.  Replaces building the whole index on every host."""
        import torch.distributed as dist

        from .index import global_bm25_stats

        def hook(term_token, df, n_docs, n_tokens):
            if self.world == 1:
                parts = [(term_token, df, n_docs, n_tokens)]
            else:
                parts = [None] * self.world
                dist.all_gather_object(parts, (np.asarray(term_token), np.asarray(df), int(n_docs), int(n_tokens)),
                                       group=self.group)
            idf_of, avg_idf, _, avgdl = global_bm25_stats([p[0] for p in parts], [p[1] for p in parts],
                                                          [p[2] for p in parts], [p[3] for p in parts], variant, epsilon)
            return idf_of, avg_idf, avgdl

        data = self.engine.build_bm25_gpu(flat_tokens, doc_offsets, variant=variant, k1=k1, b=b, epsilon=epsilon,
                                          delta=delta, id_base=id_base, export=export, stats_hook=hook)
        data.extras["shard_local"] = True   # postings / doc_len cover THIS rank's doc range only
        return data

    def load_tags(self, field: int, codes: np.ndarray) -> None:
        """Payload index column ``field`` (< 16) for filtered search.  ``codes`` is the corpus-global column: one int32
        code per global doc id from one dictionary for the whole corpus (-1 = key absent); this rank loads its own slice
        into dense slot 0 and into BM25 (whichever are loaded).  Call it after loading the indexes: installing a BM25
        index drops its columns."""
        c = np.ascontiguousarray(codes, dtype=np.int32).reshape(-1)
        n_dense = self.engine.dense_count.get(0)
        has_bm25 = self.engine.bm25 is not None
        if n_dense is None and not has_bm25:
            raise ValueError("load_tags: load the dense or BM25 index first")
        if n_dense is not None:
            self.engine.load_dense_tags(field, c[self.id_base:self.id_base + n_dense], slot=0)
        if has_bm25:
            base = self.engine.bm25_id_base
            self.engine.load_bm25_tags(field, c[base:base + self.engine.bm25_count()])

    def load_cross_encoder(self, weights) -> None:
        """weights: sentio_b200.cross_encoder.CrossEncoderWeights"""
        self.engine.ce_load(weights.blob(), weights.config)

    def load_doc_tokens(self, doc_tok: np.ndarray, doc_len: np.ndarray, id_base: int = 0) -> None:
        """Pre-tokenised documents for the rerank stage.  Sharded runs replicate the (small) token matrix on every
        rank (id_base = 0, all docs), so any global candidate id can be framed locally without a second collective."""
        self.engine.ce_tokens_load(doc_tok, doc_len, id_base)

    # ------------------------------------------------------------------ helpers
    def _buf(self, name, shape, dtype):
        t = self._bufs.get(name)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = self.torch.empty(shape, dtype=dtype, device=self._torch_device)
            self._bufs[name] = t
        return t

    def _to_dev(self, arr: np.ndarray, name: str = "in"):
        """host array -> device tensor through a cached (pinned staging, device) buffer pair per call-site name and
        shape: no allocator activity on the hot path (a fresh torch allocation per call showed 50 ms hiccups)."""
        t = self.torch.from_numpy(arr)
        if self.device is None:
            return t
        key = ("pin", name, tuple(arr.shape), arr.dtype.str)
        pair = self._bufs.get(key)
        if pair is None:
            pair = (self.torch.empty(arr.shape, dtype=t.dtype, pin_memory=True),
                    self.torch.empty(arr.shape, dtype=t.dtype, device=self._torch_device))
            self._bufs[key] = pair
        pin, dev = pair
        pin.copy_(t)
        dev.copy_(pin, non_blocking=True)
        return dev

    def _to_host(self, tensors, name: str = "out"):
        """device tensors -> NumPy arrays through cached pinned buffers: all copies are enqueued, ONE synchronisation."""
        if self.device is None:
            return tuple(t.numpy().copy() for t in tensors)   # copies: the tensors are cached buffers reused by the next call
        outs = []
        for i, t in enumerate(tensors):
            key = ("pin_out", name, i, tuple(t.shape), t.dtype)
            pin = self._bufs.get(key)
            if pin is None:
                pin = self.torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                self._bufs[key] = pin
            pin.copy_(t, non_blocking=True)
            outs.append(pin)
        self.torch.cuda.current_stream().synchronize()
        return tuple(p.numpy().copy() for p in outs)

    def _filters_to_dev(self, filters):
        """host CSR conditions (f_off, f_field, f_code) -> int32 device tensors; None stays None"""
        if filters is None:
            return None
        off, fld, code = (np.ascontiguousarray(a, dtype=np.int32).reshape(-1) for a in filters)
        if len(fld) != len(code) or int(off[-1]) != len(fld):
            raise ValueError("filters must be CSR (f_off [B+1], f_field [n], f_code [n]) with f_off[B] == n")
        return self._to_dev(off, "f_off"), self._to_dev(fld, "f_field"), self._to_dev(code, "f_code")

    def _record_layout(self, B: int, k: int, signals: int):
        """Byte layout of one rank's all-gather record: per signal ids[B,k] i64 | scores[B,k] f64 | counts[B] i32."""
        per = B * k * 8 * 2 + ((B * 4 + 7) // 8) * 8
        return per, per * signals

    def _views(self, rec, B, k, sig):
        t = self.torch
        per, _ = self._record_layout(B, k, 1)
        base = sig * per
        ids = rec[base: base + B * k * 8].view(t.int64).view(B, k)
        sc = rec[base + B * k * 8: base + B * k * 16].view(t.float64).view(B, k)
        cnt = rec[base + B * k * 16: base + B * k * 16 + B * 4].view(t.int32)
        return ids, sc, cnt

    def _gather(self, rec):
        """The single collective of the path: all-gather of the per-rank record over NCCL (NVLink/NVSwitch)."""
        import torch.distributed as dist

        out = self._buf("gathered", (self.world, rec.numel()), self.torch.uint8)
        with self._stage("all_gather_us"):
            dist.all_gather_into_tensor(out.view(-1), rec, group=self.group)
        return out

    # ------------------------------------------------------------------ optional stage timing
    class _Span:
        def __init__(self, pipe, name):
            self.pipe, self.name = pipe, name

        def __enter__(self):
            if self.pipe.stage_timing and self.pipe.device is not None:
                t = self.pipe.torch
                self.a, self.b = t.cuda.Event(enable_timing=True), t.cuda.Event(enable_timing=True)
                self.a.record()
            return self

        def __exit__(self, *exc):
            if self.pipe.stage_timing and self.pipe.device is not None:
                self.b.record()
                self.pipe._stage_events.append((self.name, self.a, self.b))
            return False

    def _stage(self, name: str):
        return HybridPipeline._Span(self, name)

    def stage_ms(self) -> dict:
        """Drains the recorded stage spans: name -> summed milliseconds (and ``stage_counts[name]`` spans)."""
        self.torch.cuda.synchronize()
        out: dict = {}
        self.stage_counts = {}
        for name, a, b in self._stage_events:
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
            self.stage_counts[name] = self.stage_counts.get(name, 0) + 1
        self._stage_events = []
        return out

    # ------------------------------------------------------------------ device-resident path
    def dense_dev(self, q_t, k: int, filters=None):
        """q_t [B,d] fp32 cuda -> global (ids, scores, counts) on this rank.  ``filters``: CSR conditions as int32 device
        tensors (f_off [B+1], f_field, f_code), applied on every shard before the merge; None = unfiltered."""
        t = self.torch
        B = q_t.shape[0]
        fkw = {} if filters is None else {"filters": filters}
        if self.world == 1:
            out = (self._buf("d_ids", (B, k), t.int64), self._buf("d_sc", (B, k), t.float64),
                   self._buf("d_cnt", (B,), t.int32))
            return self.engine.dense_topk_dev(q_t, k, out=out, **fkw)
        _, nbytes = self._record_layout(B, k, 1)
        rec = self._buf("rec1", (nbytes,), t.uint8)
        with self._stage("local_dense_topk_us"):
            self.engine.dense_topk_dev(q_t, k, out=self._views(rec, B, k, 0), **fkw)
        g = self._gather(rec)
        ids0, sc0, cnt0 = self._views(g[0], B, k, 0)
        out = (self._buf("d_ids", (B, k), t.int64), self._buf("d_sc", (B, k), t.float64),
               self._buf("d_cnt", (B,), t.int32))
        with self._stage("merge_shards_us"):
            return self.engine.merge_shards_dev(ids0, sc0, cnt0, nbytes, self.world, out=out)

    def hybrid_dev(self, q_t, terms_t, off_t, n_terms: int, max_len: int, k: int, method: str = "rrf",
                   rrf_k: float = 60, w_dense: float = 0.5, w_sparse: float = 0.5, filters=None):
        """Dense + BM25 + fusion for a batch; returns fused (ids, scores, src, counts) device tensors.  ``filters``: CSR
        conditions as int32 device tensors, applied to both signals on every shard (fusion then sees only matching
        docs); None = unfiltered."""
        t = self.torch
        B = q_t.shape[0]
        fkw = {} if filters is None else {"filters": filters}
        per, nbytes = self._record_layout(B, k, 2)
        rec = self._buf("rec2", (nbytes,), t.uint8)
        dv = self._views(rec, B, k, 0)
        sv = self._views(rec, B, k, 1)
        self.engine.dense_topk_dev(q_t, k, out=dv, **fkw)
        self.engine.bm25_topk_dev(terms_t, off_t, B, n_terms, max_len, k, out=sv, **fkw)
        if self.world > 1:
            g = self._gather(rec)
            d0 = self._views(g[0], B, k, 0)
            s0 = self._views(g[0], B, k, 1)
            dv = self.engine.merge_shards_dev(*d0, nbytes, self.world,
                                              out=(self._buf("gd_ids", (B, k), t.int64),
                                                   self._buf("gd_sc", (B, k), t.float64),
                                                   self._buf("gd_cnt", (B,), t.int32)))
            sv = self.engine.merge_shards_dev(*s0, nbytes, self.world,
                                              out=(self._buf("gs_ids", (B, k), t.int64),
                                                   self._buf("gs_sc", (B, k), t.float64),
                                                   self._buf("gs_cnt", (B,), t.int32)))
        out = (self._buf("f_ids", (B, k), t.int64), self._buf("f_sc", (B, k), t.float64),
               self._buf("f_src", (B, k), t.int32), self._buf("f_cnt", (B,), t.int32))
        return self.engine.fuse_dev(method, rrf_k, w_dense, w_sparse, k, dv, sv, out=out)

    def hybrid_rerank_dev(self, q_t, terms_t, off_t, n_terms: int, max_len: int, q_tok_t, q_len_t, k: int, k_out: int,
                          seq_len: int = 128, method: str = "rrf", rrf_k: float = 60, w_dense: float = 0.5,
                          w_sparse: float = 0.5, filters=None):
        """retrieve (dense + BM25 + fusion, top k) -> cross-encoder rerank (top k_out), all on the device.  ``filters`` as
        ``hybrid_dev``: every candidate the reranker sees matches its query's conditions.

        Sharded runs: after the all-gather + merge every rank holds the fused candidates of ALL queries; the rerank (the
        expensive stage) is then split by query -- rank r scores queries ``rerank_slice(B)`` and returns only those rows
        (no second collective; the caller owns the per-rank result slices)."""
        t = self.torch
        fkw = {} if filters is None else {"filters": filters}
        ids, sc, src, cnt = self.hybrid_dev(q_t, terms_t, off_t, n_terms, max_len, k, method, rrf_k, w_dense, w_sparse,
                                            **fkw)
        lo, hi = self.rerank_slice(q_t.shape[0])
        B = hi - lo
        out = (self._buf("r_ids", (B, k_out), t.int64), self._buf("r_sc", (B, k_out), t.float32),
               self._buf("r_cnt", (B,), t.int32))
        if B == 0:
            return out
        return self.engine.rerank_dev(q_tok_t[lo:hi], q_len_t[lo:hi], ids[lo:hi], cnt[lo:hi], seq_len, k_out, out=out)

    def rerank_slice(self, B: int):
        """[lo, hi) of the batch that this rank reranks (the whole batch on a single GPU)."""
        if self.world == 1:
            return 0, B
        per = (B + self.world - 1) // self.world
        return min(B, self.rank * per), min(B, (self.rank + 1) * per)

    # ------------------------------------------------------------------ host (e2e) path
    def search_dense(self, q: np.ndarray, k: int, out=None, filters=None):
        """Host in / host out.  world == 1: straight through the C-ABI host entry point (``out``: arrays to fill in
        place -- page-locked ones from ``engine.pinned_empty`` skip the staging copies).  ``filters``: host CSR
        conditions (f_off [B+1], f_field, f_code) int32 arrays, or None (unfiltered)."""
        if filters is not None:
            if self.world == 1:
                return self.engine.dense_topk(q, k, filters=filters)
            q_t = self._to_dev(np.ascontiguousarray(q, dtype=np.float32), "q")
            return self._to_host(self.dense_dev(q_t, k, filters=self._filters_to_dev(filters)), "dense")
        if self.world == 1:
            return self.engine.dense_topk(q, k, out=out) if out is not None else self.engine.dense_topk(q, k)
        t = self.torch
        q_t = self._to_dev(np.ascontiguousarray(q, dtype=np.float32), "q")
        return self._to_host(self.dense_dev(q_t, k), "dense")

    def search_hybrid(self, q: np.ndarray, term_lists: Sequence[Sequence[int]], k: int, method: str = "rrf",
                      rrf_k: float = 60, w_dense: float = 0.5, w_sparse: float = 0.5, filters=None):
        """Host in / host out.  ``filters``: host CSR conditions (f_off [B+1], f_field, f_code) int32 arrays applied to
        both signals (field f must be loaded for dense and BM25, see ``load_tags``), or None (unfiltered)."""
        import os
        import time

        trace = os.environ.get("SENTIO_B200_TRACE") == "1"
        t0 = time.perf_counter()
        flat, off = B200Engine.pack_queries(term_lists)
        if self.world == 1 and self.device is not None:
            # single shard: straight through the C ABI's host entry point (its own pinned staging, no framework on the path)
            if filters is not None:
                return self.engine.hybrid_topk(q, flat, off, k, method, rrf_k, w_dense, w_sparse, filters=filters)
            return self.engine.hybrid_topk(q, flat, off, k, method, rrf_k, w_dense, w_sparse)
        max_len = int(np.diff(off).max()) if len(off) > 1 else 0
        t1 = time.perf_counter()
        q_t = self._to_dev(np.ascontiguousarray(q, dtype=np.float32), "q")
        terms_t = self._to_dev(flat, "terms")
        off_t = self._to_dev(off, "off")
        fkw = {} if filters is None else {"filters": self._filters_to_dev(filters)}
        t2 = time.perf_counter()
        dev = self.hybrid_dev(q_t, terms_t, off_t, int(off[-1]), max_len, k, method, rrf_k, w_dense, w_sparse, **fkw)
        t3 = time.perf_counter()
        out = self._to_host(dev, "hybrid")
        if trace:
            t4 = time.perf_counter()
            print(f"[trace] search_hybrid B={len(term_lists)}: pack {1e3 * (t1 - t0):.3f} ms, to_dev {1e3 * (t2 - t1):.3f}, "
                  f"enqueue {1e3 * (t3 - t2):.3f}, wait+to_host {1e3 * (t4 - t3):.3f}", flush=True)
        return out

    def search_hybrid_rerank(self, q: np.ndarray, term_lists, q_tok: np.ndarray, q_len: np.ndarray, k: int, k_out: int,
                             seq_len: int = 128, method: str = "rrf", rrf_k: float = 60, w_dense: float = 0.5,
                             w_sparse: float = 0.5, filters=None):
        """``filters`` as ``search_hybrid``; a filtered call reranks through ``hybrid_rerank_dev``."""
        flat, off = B200Engine.pack_queries(term_lists)
        if self.world == 1 and self.device is not None and filters is None:  # one shard: the C ABI host entry point
            return self.engine.hybrid_rerank_topk(q, flat, off, q_tok, q_len, k, k_out, seq_len, method, rrf_k, w_dense,
                                                  w_sparse)
        max_len = int(np.diff(off).max()) if len(off) > 1 else 0
        q_t = self._to_dev(np.ascontiguousarray(q, dtype=np.float32), "q")
        terms_t, off_t = self._to_dev(flat, "terms"), self._to_dev(off, "off")
        qt_t = self._to_dev(np.ascontiguousarray(q_tok, dtype=np.int32), "qtok")
        ql_t = self._to_dev(np.ascontiguousarray(q_len, dtype=np.int32), "qlen")
        fkw = {} if filters is None else {"filters": self._filters_to_dev(filters)}
        return self._to_host(self.hybrid_rerank_dev(q_t, terms_t, off_t, int(off[-1]), max_len, qt_t, ql_t, k, k_out,
                                                    seq_len, method, rrf_k, w_dense, w_sparse, **fkw), "rerank")
