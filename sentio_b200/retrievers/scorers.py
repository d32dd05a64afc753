"""Scorer plugins (same classes / constructor arguments as reference src/core/retrievers/scorers.py:25-273).

* ``KeywordMatchScorer`` / ``RecencyScorer`` -- host-side string / timestamp work, exactly the reference formulas.
* ``SemanticSimilarityScorer`` / ``MMRScorer`` -- the cosine, Gram-matrix and greedy-selection arithmetic runs on the
  GPU (csrc/mmr.cu).  By default the candidate embeddings come from ``embedder.embed_many_sync`` like the reference;
  with ``vector_source=(store, collection)`` they are gathered from the HBM-resident corpus by document id instead,
  which removes n embedding calls per query (the reference's dominant cost, SURVEY.md section 3.2).
"""
from __future__ import annotations

import logging
import re
import time

import numpy as np

from ..document import Document
from ..engine import B200Engine

__all__ = ["KeywordMatchScorer", "MMRScorer", "RecencyScorer", "SemanticSimilarityScorer"]

logger = logging.getLogger(__name__)
_WORD = re.compile(r"\w+")

_shared_engine: B200Engine | None = None


def _engine(device: int = 0) -> B200Engine:
    global _shared_engine
    if _shared_engine is None:
        _shared_engine = B200Engine(device)
    return _shared_engine


class KeywordMatchScorer:
    """``weight * |keywords(query) & words(doc)| / |keywords(query)|`` with ``\\w+`` word extraction."""

    def __init__(self, weight: float = 0.5, case_sensitive: bool = False):
        self.weight = weight
        self.case_sensitive = case_sensitive

    def score(self, query: str, docs: list[Document]) -> list[float]:
        keywords = set(_WORD.findall(query.lower()))
        if not keywords:
            return [0.0] * len(docs)
        out = []
        for doc in docs:
            text = doc.text if self.case_sensitive else doc.text.lower()
            matches = len(keywords & set(_WORD.findall(text)))
            out.append((matches / len(keywords)) * self.weight)
        return out


class RecencyScorer:
    """``(1 - min(age, max_age) / max_age) * weight`` for numeric ``metadata[timestamp_field]`` not in the future."""

    def __init__(self, timestamp_field: str = "timestamp", weight: float = 0.3, max_age_seconds: int = 86400 * 30):
        self.timestamp_field = timestamp_field
        self.weight = weight
        self.max_age_seconds = max_age_seconds

    def score(self, query: str, docs: list[Document]) -> list[float]:
        now = time.time()
        out = []
        for doc in docs:
            value = 0.0
            ts = doc.metadata.get(self.timestamp_field)
            if ts and isinstance(ts, (int, float)):
                age = now - ts
                if age >= 0:
                    value = (1 - min(age, self.max_age_seconds) / self.max_age_seconds) * self.weight
            out.append(value)
        return out


class _GpuEmbeddingScorer:
    def __init__(self, embedder, engine: B200Engine | None, vector_source, device: int):
        self.embedder = embedder
        self._engine = engine
        self._vector_source = vector_source  # (B200VectorStore, collection_name) or None
        self._device = device

    def _semantic_mmr(self, query: str, docs: list[Document], **kw):
        """``semantic_mmr`` of the query against the docs: their stored rows when every doc id is in the vector source,
        else their re-embedded texts."""
        q = np.asarray(self.embedder.embed_sync(query), dtype=np.float32)
        if self._vector_source is not None:
            store, collection = self._vector_source
            # the id -> row lookup and the device call under one hold of the collection's lock: an upsert / delete in
            # between moves rows, and a row looked up before it would score another point's vector
            with store.locked(collection):
                rows = store.rows_of(collection, [d.id for d in docs])
                if (rows >= 0).all():
                    return store.engine_of(collection).semantic_mmr(q, cand_ids=rows, **kw)
        cand = np.asarray(self.embedder.embed_many_sync([d.text for d in docs]), dtype=np.float32)
        return (self._engine or _engine(self._device)).semantic_mmr(q, cand=cand, **kw)


class SemanticSimilarityScorer(_GpuEmbeddingScorer):
    """``weight * cos(query, doc)``; zeros when a norm is zero; zeros for every doc on any failure."""

    def __init__(self, embedder, weight: float = 0.7, engine: B200Engine | None = None, vector_source=None,
                 device: int = 0):
        super().__init__(embedder, engine, vector_source, device)
        self.weight = weight

    def score(self, query: str, docs: list[Document]) -> list[float]:
        try:
            if not docs:
                return []
            sem, _ = self._semantic_mmr(query, docs, w_sem=self.weight, want_sem=True, want_mmr=False)
            return [float(x) for x in sem]
        except Exception as exc:
            logger.warning("Error in semantic scoring: %s", exc)
            return [0.0] * len(docs)


class MMRScorer(_GpuEmbeddingScorer):
    """Greedy maximal-marginal-relevance scores, ``lambda * relevance - (1 - lambda) * max-redundancy`` (times weight)."""

    def __init__(self, embedder, lambda_: float = 0.7, weight: float = 0.5, engine: B200Engine | None = None,
                 vector_source=None, device: int = 0):
        if not 0.0 <= lambda_ <= 1.0:
            raise ValueError("lambda_ must be between 0 and 1 inclusive")
        super().__init__(embedder, engine, vector_source, device)
        self.lambda_ = lambda_
        self.weight = weight

    def score(self, query: str, docs: list[Document]) -> list[float]:
        if not docs:
            return []
        try:
            _, mmr = self._semantic_mmr(query, docs, lambda_=self.lambda_, w_mmr=self.weight, want_sem=False,
                                        want_mmr=True)
            return [float(x) for x in mmr]
        except Exception as exc:
            logger.warning("MMR scorer failed: %s", exc)
            return [0.0] * len(docs)
