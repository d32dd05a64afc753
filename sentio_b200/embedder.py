"""B200Embedder -- query / document embeddings from an encoder that runs on the GPU (SURVEY.md §8f row 1).

The step immediately before the dense search in ``DenseRetriever.retrieve`` is ``self.embedder.embed_sync(query)``
(reference src/core/retrievers/dense.py:43), a remote call to the Jina embeddings API in the reference
(src/core/embeddings/providers/jina.py).  This class has the surface of the reference's ``BaseEmbedder``
(src/core/embeddings/base.py:146-420: ``embed_sync`` / ``embed_many_sync`` / ``embed_async_single`` /
``embed_async_many`` / ``dimension`` / ``stats`` / ``warm_up`` / ``close``, LFU-free dict cache) and computes the
embedding locally: hashed word pieces ``[CLS] tokens [SEP]`` -> BERT-style encoder (the cross-encoder's kernels:
wgmma GEMMs, packed tokens, [CLS]-only last layer) -> optional linear projection to ``dimension`` -> L2 normalise.

There is no checkpoint offline, so the weights are random-init (MiniLM-L6 shape + a 384 -> 1024 projection by default,
matching the 1024-d vectors of BASELINE.json); parity is against the HuggingFace ``BertModel`` forward of the same
weights (tests/test_embedder_gpu.py).
"""
from __future__ import annotations

import logging

import asyncio
import time
from typing import Any

import numpy as np

from .cross_encoder import MINILM_L6, CrossEncoderWeights
from .index import CLS_ID, PAD_ID, SEP_ID, _hash_token


def tokenize_for_embedding(texts, seq_len: int = 128):
    """``[CLS] hashed-word-pieces [SEP]`` (crc32 hash, sentio_b200.index) padded / truncated to ``seq_len``."""
    P = len(texts)
    ids = np.full((P, seq_len), PAD_ID, dtype=np.int32)
    tt = np.zeros((P, seq_len), dtype=np.int32)
    lens = np.zeros(P, dtype=np.int32)
    for i, text in enumerate(texts):
        toks = [_hash_token(t) for t in (text or "").lower().split()][: seq_len - 2]
        row = [CLS_ID, *toks, SEP_ID]
        ids[i, :len(row)] = row
        lens[i] = len(row)
    return ids, tt, lens


logger = logging.getLogger(__name__)


class B200Embedder:
    def __init__(self, model_name: str = "b200-minilm-l6-random", weights: CrossEncoderWeights | None = None,
                 proj_w: np.ndarray | None = None, proj_b: np.ndarray | None = None, dimension: int = 1024,
                 seq_len: int = 128, device: int = 0, engine=None, cache_enabled: bool = True, cache_size: int = 10_000,
                 seed: int = 0, allow_random_init: bool = False, **kwargs: Any) -> None:
        """``weights`` are required (no checkpoint ships offline): ``allow_random_init=True`` builds the random-init
        MiniLM-L6 encoder the tests and benchmarks use -- its embeddings are well formed and meaningless."""
        self.model_name = model_name
        self.seq_len = int(seq_len)
        self._cache_enabled = cache_enabled
        self._cache: dict[str, list[float]] = {}
        self._cache_size = int(cache_size)
        self._stats = {"total_requests": 0, "cache_hits": 0, "errors": 0, "total_time": 0.0}
        if weights is None:
            if not allow_random_init:
                raise ValueError("B200Embedder needs weights=CrossEncoderWeights(...); pass allow_random_init=True only "
                                 "for tests / benchmarks")
            logger.warning("B200Embedder: RANDOM-INIT encoder weights (seed %d) -- embeddings are meaningless", seed)
            weights = CrossEncoderWeights.random(MINILM_L6, seed=seed)
        hidden = int(weights.config["hidden"])
        if proj_w is None and dimension != hidden:
            rng = np.random.default_rng(seed + 1)
            proj_w = (rng.standard_normal((dimension, hidden), dtype=np.float32) / np.float32(np.sqrt(hidden)))
            proj_b = np.zeros(dimension, dtype=np.float32)
        self.weights, self.proj_w, self.proj_b = weights, proj_w, proj_b
        if engine is None:
            from .engine import B200Engine

            engine = B200Engine(device)
        self._engine = engine
        engine.enc_load(weights.blob(), weights.config, proj_w, proj_b)
        self._dimension = engine.enc_dim()

    # ------------------------------------------------------------------ BaseEmbedder surface
    @property
    def dimension(self) -> int:
        return self._dimension

    @property
    def stats(self) -> dict[str, Any]:
        s = dict(self._stats)
        s["avg_time"] = s["total_time"] / s["total_requests"] if s["total_requests"] else 0.0
        s["cache_size"] = len(self._cache)
        return s

    def reset_stats(self) -> None:
        self._stats = {"total_requests": 0, "cache_hits": 0, "errors": 0, "total_time": 0.0}

    def embed_arrays(self, texts: list[str]) -> np.ndarray:
        """[len(texts), dimension] float32, one GPU batch."""
        ids, tt, lens = tokenize_for_embedding(texts, self.seq_len)
        return self._engine.enc_embed(ids, tt, lens, normalize=True)

    def embed_many_sync(self, texts: list[str]) -> list[list[float]]:
        t0 = time.perf_counter()
        out: list[list[float] | None] = [None] * len(texts)
        todo = []
        for i, t in enumerate(texts):
            hit = self._cache.get(t) if self._cache_enabled else None
            if hit is not None:
                out[i] = hit
                self._stats["cache_hits"] += 1
            else:
                todo.append(i)
        if todo:
            try:
                vecs = self.embed_arrays([texts[i] for i in todo])
            except Exception:
                self._stats["errors"] += 1
                raise
            for i, v in zip(todo, vecs):
                lst = [float(x) for x in v]
                out[i] = lst
                if self._cache_enabled and len(self._cache) < self._cache_size:
                    self._cache[texts[i]] = lst
        self._stats["total_requests"] += len(texts)
        self._stats["total_time"] += time.perf_counter() - t0
        return out  # type: ignore[return-value]

    def embed_sync(self, text: str) -> list[float]:
        return self.embed_many_sync([text])[0]

    async def embed_async_single(self, text: str) -> list[float]:
        return await asyncio.get_running_loop().run_in_executor(None, self.embed_sync, text)

    async def embed_async_many(self, texts: list[str]) -> list[list[float]]:
        return await asyncio.get_running_loop().run_in_executor(None, self.embed_many_sync, texts)

    async def warm_up(self, sample_texts: list[str] | None = None) -> bool:
        try:
            await self.embed_async_many(sample_texts or ["warm up"])
            return True
        except Exception:
            return False

    async def close(self) -> None:
        self._cache.clear()
