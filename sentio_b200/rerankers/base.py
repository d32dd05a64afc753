"""Reranker interfaces of the GPU path.

``create_reranker_node`` (reference src/core/graph/nodes.py:124-127,179-183) calls ``reranker.rerank(query=, docs=,
top_k=)`` and nothing else; ``rerank_async`` and the ``RerankingResult`` container complete the surface of the reference's
src/core/rerankers/base.py:14-132.  ``rerank_batch`` is the addition of this package: many (query, candidate list) jobs in
one call, which a GPU cross-encoder turns into a single forward pass over all pairs.
"""
from __future__ import annotations

import abc
import asyncio
import functools
from dataclasses import dataclass, field
from typing import Any, Iterator, Protocol, Sequence

from ..document import Document

__all__ = ["Reranker", "RerankerProtocol", "RerankingResult"]


class RerankerProtocol(Protocol):
    """Structural type of anything the reranker node accepts."""

    def rerank(self, query: str, docs: list[Document], top_k: int = 5, **kwargs: Any) -> list[Document]: ...

    async def rerank_async(self, query: str, docs: list[Document], top_k: int = 5, **kwargs: Any) -> list[Document]: ...


@dataclass
class RerankingResult:
    """Reranked documents plus the originals and free-form metadata; behaves like a sequence over ``documents``."""

    documents: list[Document]
    original_documents: list[Document] = field(default_factory=list)
    metadata: dict[str, Any] = field(default_factory=dict)

    def __post_init__(self) -> None:  # the reference accepts None for both optional arguments
        self.original_documents = self.original_documents or []
        self.metadata = self.metadata or {}

    @property
    def top_document(self) -> Document | None:
        return self.documents[0] if self.documents else None

    def __len__(self) -> int:
        return len(self.documents)

    def __getitem__(self, idx: int) -> Document:
        return self.documents[idx]

    def __iter__(self) -> Iterator[Document]:
        return iter(self.documents)


class Reranker(abc.ABC):
    """Abstract reranker: ``rerank`` is the one method a subclass must provide."""

    @abc.abstractmethod
    def rerank(self, query: str, docs: list[Document], top_k: int = 5, **kwargs: Any) -> list[Document]:
        """``docs`` reordered by relevance to ``query`` (best first), truncated to ``top_k``."""
        raise NotImplementedError

    def rerank_batch(self, queries: Sequence[str], docs_per_query: Sequence[list[Document]], top_k: int = 5,
                     **kwargs: Any) -> list[list[Document]]:
        """One reranked list per (query, candidate list) job.  Default: a loop over ``rerank``."""
        if len(queries) != len(docs_per_query):
            raise ValueError("queries and docs_per_query must have the same length")
        return [self.rerank(q, d, top_k=top_k, **kwargs) for q, d in zip(queries, docs_per_query)]

    async def rerank_async(self, query: str, docs: list[Document], top_k: int = 5, **kwargs: Any) -> list[Document]:
        """``rerank`` on the event loop's default executor."""
        job = functools.partial(self.rerank, query, docs, top_k, **kwargs)
        return await asyncio.get_running_loop().run_in_executor(None, job)
