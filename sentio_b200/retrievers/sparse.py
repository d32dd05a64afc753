"""BM25Retriever -- BM25 Okapi / Plus over GPU-resident CSR postings (K2).

Same surface as reference src/core/retrievers/sparse.py:33-203: ``BM25Retriever(documents=None, variant="okapi",
cache_dir=None)``, ``index``, ``save``, ``load``, ``retrieve``; tokeniser ``text.lower().split()``; ``BM25_VARIANT`` /
``SPARSE_CACHE_DIR`` environment overrides; results are the corpus ``Document`` objects themselves with
``metadata["bm25_score"]`` written in place; scores <= 0 are dropped; any failure returns ``[]``.

Deviation (documented in DESIGN.md): ties are ordered (score desc, corpus position asc) -- the reference's
``np.argsort(-scores)`` is an unstable introsort whose tie order is implementation defined.
"""
from __future__ import annotations

import logging
import os
import pickle

import numpy as np

from ..document import Document
from ..engine import B200Engine
from ..index import Bm25IndexData, tokenize_texts
from .base import BaseRetriever

logger = logging.getLogger(__name__)

_SAVE_FORMAT = "sentio_b200.bm25retriever.v1"
_KERNEL_MAX_K = 1024  # top-k limit of one sb_bm25_topk call (shared-memory winner buffer, bm25.cu)


class BM25Retriever(BaseRetriever):
    def __init__(self, documents: list[Document] | None = None, variant: str = "okapi", cache_dir: str | None = None,
                 device: int = 0, k1: float = 1.5, b: float = 0.75, epsilon: float = 0.25, delta: float = 1.0):
        self.bm25: Bm25IndexData | None = None  # the name the reference uses for its rank_bm25 object
        self.doc_ids: list[str] = []
        self.doc_map: dict[str, Document] = {}
        self.tokenized_corpus: list[list[str]] = []
        self.variant = os.environ.get("BM25_VARIANT", variant).lower()
        self.cache_dir = cache_dir or os.environ.get("SPARSE_CACHE_DIR", ".sparse_cache")
        self._params = dict(k1=k1, b=b, epsilon=epsilon, delta=delta)
        self._device = device
        self._engine: B200Engine | None = None
        if documents:
            self.index(documents)

    # ------------------------------------------------------------------ build / persist
    def _upload(self) -> None:
        if self._engine is None:
            self._engine = B200Engine(self._device)
        self._engine.load_bm25(self.bm25, id_base=0)

    def index(self, documents: list[Document]) -> None:
        if not documents:
            logger.warning("Empty document list provided for BM25 indexing")
            return
        self.doc_ids = [doc.id for doc in documents]
        self.doc_map = {doc.id: doc for doc in documents}
        variant = "plus" if self.variant == "plus" else "okapi"
        # strings -> first-occurrence token ids on the host (sparse.py:88's tokeniser); everything numeric -- sort, df,
        # tf, CSR -- on the device (sb_bm25_build_*); the CSR is exported once so save() / load() keep working
        vocab, flat, off = tokenize_texts(doc.text for doc in documents)
        if len(flat) == 0:
            logger.warning("BM25 corpus has no tokens")
            return
        if self._engine is None:
            self._engine = B200Engine(self._device)
        self.bm25 = self._engine.build_bm25_gpu(flat, off, variant=variant, id_base=0, export=True, **self._params)
        self.bm25.vocab = vocab
        self.bm25.token_id_map = None
        self.tokenized_corpus = []  # not retained: the CSR index replaces it (reconstruct lazily if ever needed)
        logger.info("BM25 (%s) index on GPU: %d docs, %d terms, %d postings", variant, self.bm25.n_docs,
                    self.bm25.n_terms, len(self.bm25.post_doc))

    def save(self, filepath: str | None = None) -> None:
        if not self.bm25:
            logger.warning("Cannot save empty BM25 index")
            return
        if not filepath:
            os.makedirs(self.cache_dir, exist_ok=True)
            filepath = os.path.join(self.cache_dir, "bm25_index.pkl")
        try:
            with open(filepath, "wb") as f:
                pickle.dump({"format": _SAVE_FORMAT, "bm25": self.bm25, "doc_ids": self.doc_ids,
                             "doc_map": self.doc_map, "variant": self.variant}, f, protocol=pickle.HIGHEST_PROTOCOL)
        except Exception as exc:  # same contract as the reference: log, do not raise
            logger.error("Failed to save BM25 index: %s", exc)

    def load(self, filepath: str | None = None) -> bool:
        if not filepath:
            filepath = os.path.join(self.cache_dir, "bm25_index.pkl")
        try:
            if not os.path.exists(filepath):
                logger.warning("BM25 index file not found: %s", filepath)
                return False
            with open(filepath, "rb") as f:
                data = pickle.load(f)
            # validate into locals first: a foreign pickle (e.g. the reference's rank_bm25 cache) or a failed upload
            # must leave the retriever exactly as it was
            if not isinstance(data, dict) or data.get("format") != _SAVE_FORMAT:
                raise ValueError(f"{filepath} is not a {_SAVE_FORMAT} file")
            bm25, doc_ids = data["bm25"], list(data["doc_ids"])
            if not isinstance(bm25, Bm25IndexData) or len(doc_ids) != int(bm25.n_docs):
                raise ValueError("BM25 index payload is inconsistent")
            if self._engine is None:
                self._engine = B200Engine(self._device)
            self._engine.load_bm25(bm25, id_base=0)
            self.bm25, self.doc_ids = bm25, doc_ids
            self.doc_map = data.get("doc_map", {})
            self.variant = data.get("variant", "okapi")
            return True
        except Exception as exc:
            logger.error("Failed to load BM25 index: %s", exc)
            return False

    # ------------------------------------------------------------------ query
    def retrieve(self, query: str, top_k: int = 10) -> list[Document]:
        if not self.bm25 or self._engine is None:
            logger.warning("BM25 index not initialized")
            return []
        try:
            ids, scores, counts = self.retrieve_batch_arrays([query], int(top_k))
            results = []
            for j in range(int(counts[0])):
                row = int(ids[0, j])
                doc_id = self.doc_ids[row]
                doc = self.doc_map.get(doc_id)
                if doc is None:
                    doc = Document(id=doc_id, text="")
                doc.metadata["bm25_score"] = float(scores[0, j])
                results.append(doc)
            return results
        except Exception as exc:
            logger.error("BM25 retrieval error: %s", exc)
            return []

    def retrieve_batch(self, queries, top_k: int = 10) -> list[list[Document]]:
        """Many queries in ONE device batch; per query the same ids, order and ``bm25_score`` as ``retrieve``.

        ``retrieve`` hands out the shared corpus objects and overwrites their ``bm25_score`` (sparse.py:189-197); a batch
        cannot do that -- the same document may be a hit of several queries -- so every hit here is a COPY of the corpus
        document carrying its own score."""
        queries = list(queries)
        if not self.bm25 or self._engine is None:
            logger.warning("BM25 index not initialized")
            return [[] for _ in queries]
        if not queries:
            return []
        try:
            ids, scores, counts = self.retrieve_batch_arrays(queries, top_k)
            out = []
            for b in range(len(queries)):
                results = []
                for j in range(int(counts[b])):
                    doc_id = self.doc_ids[int(ids[b, j])]
                    src = self.doc_map.get(doc_id)
                    meta = dict(src.metadata) if src is not None and src.metadata else {}
                    meta["bm25_score"] = float(scores[b, j])
                    results.append(Document(id=doc_id, text=src.text if src is not None else "", metadata=meta))
                out.append(results)
            return out
        except Exception as exc:
            logger.error("BM25 batch retrieval error: %s", exc)
            return [[] for _ in queries]

    def retrieve_batch_arrays(self, queries: list[str], top_k: int):
        """Batched extension: (rows, scores, counts) arrays for many queries in one GPU batch."""
        terms = [self.bm25.term_ids(q.lower().split()) for q in queries]
        k = int(top_k)
        if k <= 0:
            B = len(queries)
            return np.zeros((B, 0), np.int64), np.zeros((B, 0)), np.zeros(B, np.int32)
        k = min(k, int(self.bm25.n_docs))   # the reference's argsort[:top_k] never returns more than the corpus
        if k <= _KERNEL_MAX_K:
            return self._engine.bm25_topk(terms, k)
        # top_k beyond one kernel call (the reference supports any top_k): the device scores every document
        # (sb_bm25_scores, the same bit-exact fp64 kernel), the cut is the reference's own expression (sparse.py:180-184)
        ids = np.full((len(terms), k), -1, np.int64)
        sc = np.zeros((len(terms), k))
        cnt = np.zeros(len(terms), np.int32)
        for b, t in enumerate(terms):
            scores = self._engine.bm25_scores(t)
            order = np.argsort(-scores, kind="stable")[:k]
            order = order[scores[order] > 0]
            ids[b, :len(order)], sc[b, :len(order)], cnt[b] = order, scores[order], len(order)
        return ids, sc, cnt


class PyseriniBM25Retriever(BaseRetriever):
    """Surface of the reference's Lucene-backed retriever (sparse.py:206-276), GPU-backed.

    The reference class needs Pyserini (a JVM) and an on-disk Lucene index; without them its constructor raises
    ``RuntimeError`` and ``create_retriever_from_env`` falls back to the in-memory ``BM25Retriever`` (factory.py:150-163).
    Neither exists offline, so parity with Lucene's scorer (its lossy norm encoding, analyzers and idf form) cannot be
    pinned and is not claimed.  What this class provides is the same constructor contract -- ``index_dir`` must exist,
    else ``RuntimeError`` -- and, when given the corpus explicitly, the Pyserini DEFAULT PARAMETERS (k1 = 0.9, b = 0.4,
    ``BM25_K1`` / ``BM25_B`` in the factory) on the GPU Okapi kernel: ``PyseriniBM25Retriever(documents=docs)``.
    """

    def __init__(self, index_dir: str | None = None, k1: float = 0.9, b: float = 0.4,
                 documents: list[Document] | None = None, device: int = 0):
        self.index_dir = index_dir or os.getenv("BM25_INDEX_DIR", "indexes/lucene-index")
        if documents is None:
            if not os.path.isdir(self.index_dir):
                raise RuntimeError(f"Pyserini index directory not found: {self.index_dir}")
            raise RuntimeError("Pyserini is not installed - Lucene indexes cannot be read by the GPU path; pass "
                               "documents=... to score them with Pyserini's parameters on the GPU")
        self._inner = BM25Retriever(documents=documents, variant="okapi", device=device, k1=k1, b=b)

    def retrieve(self, query: str, top_k: int = 10) -> list[Document]:
        return self._inner.retrieve(query, top_k=top_k)
