"""Retriever / scorer interfaces of the GPU path.

The LangGraph nodes of the reference only need two things from a retriever (src/core/graph/nodes.py:37-40,70):
``retrieve(query, top_k=...)`` returning documents best first, and -- for the async graph -- ``retrieve_async``.  Both are
kept with the reference's names and defaults (src/core/retrievers/base.py:13-42) so the classes here drop into
``create_retriever_node`` / ``GraphConfig(retriever=...)`` unchanged.  On top of that every GPU-backed retriever can answer
MANY queries per call (``retrieve_batch``): one HBM pass of the dense scan serves 256 queries, so batching is where the
throughput is.
"""
from __future__ import annotations

import abc
import asyncio
from concurrent.futures import Executor
from typing import Protocol, Sequence, runtime_checkable

from ..document import Document

__all__ = ["BaseRetriever", "ScorerPlugin"]


@runtime_checkable
class ScorerPlugin(Protocol):
    """Extra scoring signal of ``HybridRetriever`` (hybrid.py:275-285): one float per document, in document order."""

    def score(self, query: str, docs: list[Document]) -> list[float]: ...


class BaseRetriever(abc.ABC):
    """Abstract retriever.  Subclasses implement ``retrieve``; the batch and async forms have working defaults."""

    #: executor used by ``retrieve_async`` (None = the event loop's default thread pool, like the reference)
    executor: Executor | None = None

    @abc.abstractmethod
    def retrieve(self, query: str, top_k: int = 10) -> list[Document]:
        """Documents for ``query``, best first, at most ``top_k``."""
        raise NotImplementedError

    def retrieve_batch(self, queries: Sequence[str], top_k: int = 10) -> list[list[Document]]:
        """One result list per query.  Default: a loop over ``retrieve``; GPU retrievers override it with a single
        batched device call."""
        return [self.retrieve(q, top_k=top_k) for q in queries]

    async def retrieve_async(self, query: str, top_k: int = 10) -> list[Document]:
        """``retrieve`` on a worker thread (the ctypes calls release the GIL, so concurrent requests overlap)."""
        return await asyncio.get_running_loop().run_in_executor(self.executor, self.retrieve, query, top_k)
