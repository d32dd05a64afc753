"""B200VectorStore -- an HBM-resident stand-in for the slice of ``qdrant_client.QdrantClient`` the hot path uses.

The reference's dense path is ``client.search(collection_name=, query_vector=, limit=, with_payload=True)``
(src/core/retrievers/dense.py:46-64), its cache probe ``client.collection_exists(collection_name=)``
(src/core/retrievers/hybrid.py:101-105) and its BM25 corpus load ``client.scroll(...)``
(src/core/retrievers/factory.py:95-101).  This class answers exactly those calls from a ``B200Engine``: vectors live in
HBM as fp16 rows (one engine per collection), payloads / ids stay on the host.  Because it is call-compatible, the
reference's OWN ``DenseRetriever`` runs unchanged on top of it (INTEGRATION.md), and so does ours.

Payload / id schema follows what the reference's ingest writes: ``payload = {"content": text, "metadata": {...}}``,
point id = string (src/core/vector_store/qdrant_store.py:333-340).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Sequence

import numpy as np

from .engine import B200Engine
from .payload_filter import PayloadIndex

__all__ = ["B200VectorStore", "ScoredPoint", "Record"]


@dataclass
class ScoredPoint:
    id: Any
    score: float
    payload: dict | None = None
    vector: Any = None
    version: int = 0


@dataclass
class Record:
    id: Any
    payload: dict | None = None
    vector: Any = None


class _Collection:
    def __init__(self, name: str, device: int):
        self.name = name
        self.engine = B200Engine(device)
        self.ids: list[Any] = []
        self.payloads: list[dict] = []
        self.row_of: dict[Any, int] = {}
        self.dim = 0
        self._payload_index: PayloadIndex | None = None

    def payload_index(self) -> PayloadIndex:
        # built lazily: a tag column per payload key, on the first filter that names the key
        if self._payload_index is None:
            self._payload_index = PayloadIndex(self.payloads,
                                               lambda f, codes: self.engine.load_dense_tags(f, codes, slot=0))
        return self._payload_index


class B200VectorStore:
    def __init__(self, device: int = 0):
        self._device = device
        self._collections: dict[str, _Collection] = {}

    # ------------------------------------------------------------------ collection management
    def collection_exists(self, collection_name: str) -> bool:
        return collection_name in self._collections

    def create_collection(self, collection_name: str, vectors: np.ndarray, ids: Sequence[Any] | None = None,
                          payloads: Sequence[dict] | None = None) -> None:
        """Upload a whole collection (brute-force search needs no incremental index)."""
        vecs = np.asarray(vectors)
        n = vecs.shape[0]
        col = _Collection(collection_name, self._device)
        col.engine.load_dense(vecs, id_base=0, slot=0)
        col.ids = list(ids) if ids is not None else [str(i) for i in range(n)]
        col.payloads = list(payloads) if payloads is not None else [{} for _ in range(n)]
        if len(col.ids) != n or len(col.payloads) != n:
            raise ValueError("ids / payloads length must match the number of vectors")
        col.row_of = {pid: i for i, pid in enumerate(col.ids)}
        col.dim = vecs.shape[1]
        old = self._collections.pop(collection_name, None)
        if old is not None:
            old.engine.close()
        self._collections[collection_name] = col

    def delete_collection(self, collection_name: str) -> None:
        col = self._collections.pop(collection_name, None)
        if col is not None:
            col.engine.close()

    def engine_of(self, collection_name: str) -> B200Engine:
        return self._collections[collection_name].engine

    def rows_of(self, collection_name: str, ids: Sequence[Any]) -> np.ndarray:
        col = self._collections[collection_name]
        return np.asarray([col.row_of.get(i, -1) for i in ids], dtype=np.int64)

    def count(self, collection_name: str) -> int:
        return len(self._collections[collection_name].ids)

    # ------------------------------------------------------------------ the calls the hot path makes
    def search(self, collection_name: str, query_vector, limit: int = 10, with_payload: bool = True,
               with_vectors: bool = False, query_filter=None, **_ignored) -> list[ScoredPoint]:
        """``query_filter``: a Qdrant ``Filter(must=[FieldCondition(key, match=MatchValue(value))...])`` or a bare
        ``FieldCondition`` (what the reference's ``_convert_filter`` emits): the exact top-``limit`` of the points whose
        payload satisfies every condition.  Other filter shapes raise ``ValueError`` (sentio_b200/payload_filter.py)."""
        col = self._collections.get(collection_name)
        if col is None:
            raise ValueError(f"Collection {collection_name} not found")
        if isinstance(query_vector, tuple):  # ("name", vector) form of the named-vector API
            query_vector = query_vector[1]
        q = np.asarray(query_vector, dtype=np.float32).reshape(1, -1)
        limit = max(1, min(int(limit), max(len(col.ids), 1)))   # Qdrant never returns more points than the collection holds
        filters = self._compile_filters(col, [query_filter]) if query_filter is not None else None
        ids, scores, counts = col.engine.dense_topk(q, int(limit), filters=filters) if filters is not None \
            else col.engine.dense_topk(q, int(limit))
        out = []
        for j in range(int(counts[0])):
            row = int(ids[0, j])
            out.append(ScoredPoint(id=col.ids[row], score=float(scores[0, j]),
                                   payload=col.payloads[row] if with_payload else None))
        return out

    def search_batch(self, collection_name: str, query_vectors, limit: int = 10, with_payload: bool = True,
                     query_filter=None, **_ignored) -> list[list[ScoredPoint]]:
        """``search`` for many query vectors in ONE device batch (the wgmma scan serves 256 queries per HBM pass).
        ``query_filter``: one filter for the whole batch, or a list / tuple with one filter (or None) per query."""
        col = self._collections.get(collection_name)
        if col is None:
            raise ValueError(f"Collection {collection_name} not found")
        q = np.asarray(query_vectors, dtype=np.float32)
        if q.ndim != 2:
            raise ValueError("query_vectors must be [B, d]")
        if q.shape[0] == 0:
            return []
        filters = None
        if query_filter is not None:
            per_query = list(query_filter) if isinstance(query_filter, (list, tuple)) else [query_filter] * q.shape[0]
            if len(per_query) != q.shape[0]:
                raise ValueError(f"query_filter: {len(per_query)} filters for {q.shape[0]} queries")
            if any(f is not None for f in per_query):
                filters = self._compile_filters(col, per_query)
        ids, scores, counts = col.engine.dense_topk(q, int(limit), filters=filters) if filters is not None \
            else col.engine.dense_topk(q, int(limit))
        return [[ScoredPoint(id=col.ids[int(ids[b, j])], score=float(scores[b, j]),
                             payload=col.payloads[int(ids[b, j])] if with_payload else None)
                 for j in range(int(counts[b]))] for b in range(q.shape[0])]

    @staticmethod
    def _compile_filters(col: _Collection, filters):
        """CSR conditions for the engine, or None when no query has a condition (the unfiltered search)."""
        off, fld, code = col.payload_index().compile(filters)
        return (off, fld, code) if len(fld) else None

    def search_batch_arrays(self, collection_name: str, query_vectors: np.ndarray, limit: int):
        """Batched extension: (rows [B,k] int64, scores [B,k] float64, counts [B]) without Python objects."""
        col = self._collections[collection_name]
        return col.engine.dense_topk(np.asarray(query_vectors, dtype=np.float32), int(limit))

    def scroll(self, collection_name: str, limit: int = 100, offset: int | None = None, with_payload: bool = True,
               with_vectors: bool = False, **_ignored):
        col = self._collections.get(collection_name)
        if col is None:
            raise ValueError(f"Collection {collection_name} not found")
        start = int(offset or 0)
        stop = min(len(col.ids), start + int(limit))
        recs = [Record(id=col.ids[i], payload=col.payloads[i] if with_payload else None) for i in range(start, stop)]
        return recs, (stop if stop < len(col.ids) else None)

    def close(self) -> None:
        for col in self._collections.values():
            col.engine.close()
        self._collections.clear()
