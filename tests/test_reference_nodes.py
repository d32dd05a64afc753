"""The reference's OWN LangGraph node functions (src/core/graph/nodes.py:37-227) driving this repository's retriever /
reranker classes -- north_star's acceptance sentence ("so the LangGraph nodes ... call it unchanged") as a test.

tests/golden/reference_nodes.json holds what the unmodified retriever node (with and without metadata.user_top_k) and
reranker node returned when they drove these classes on the oracle-backed engine double (tests/golden/make_golden.py).
The classes must still produce exactly that -- on the engine double and on the real engine / C ABI.
"""
import threading

import numpy as np
import pytest

from conftest import load_golden
from helpers import HashEmbedder
from sentio_b200.cross_encoder import CrossEncoderWeights
from sentio_b200.document import Document
from sentio_b200.rerankers.b200_reranker import B200Reranker
from sentio_b200.retrievers.dense import DenseRetriever
from sentio_b200.retrievers.hybrid import HybridRetriever

DIM = 48
TEXTS = [f"topic{i % 9} w{i % 13} w{(i * 7) % 31} alpha{i % 5} chunk number {i}" for i in range(240)]
IDS = [f"doc-{i}" for i in range(len(TEXTS))]
QUERIES = ["topic3 w4 alpha2", "w7 chunk", "nothing-in-the-vocabulary", "topic8 topic8 w30"]
CE_CFG = dict(vocab_size=30522, hidden=128, layers=2, heads=4, intermediate=256, max_pos=64, type_vocab=2, ln_eps=1e-12)


def _build(make_store, make_sparse, engine):
    emb = HashEmbedder(DIM)
    vecs = np.asarray(emb.embed_many_sync(TEXTS), dtype=np.float32)
    payloads = [{"content": t, "metadata": {"source": f"s{i % 4}", "page": i}} for i, t in enumerate(TEXTS)]
    store = make_store(vecs, IDS, payloads)
    corpus = [Document(id=i, text=t, metadata={"source": "corpus"}) for i, t in zip(IDS, TEXTS)]
    dense = DenseRetriever(client=store, embedder=emb, collection_name="Sentio_docs")
    hr = HybridRetriever(dense_retriever=dense, sparse_retriever=make_sparse(corpus), rrf_k=60, scorer_plugins=[],
                         fusion_method="rrf", engine=engine)
    rr = B200Reranker(weights=CrossEncoderWeights.random(CE_CFG, seed=3), engine=engine, seq_len=48)
    return hr, rr


def build_host_stack():
    """The classes on the oracle-backed engine double (also used by tests/golden/make_golden.py)."""
    from oracle_engine import OracleEngine
    from sentio_b200.retrievers import sparse as sparse_mod
    from test_hybrid_e2e import _OracleStore

    saved = sparse_mod.B200Engine
    sparse_mod.B200Engine = lambda device=0: OracleEngine()
    try:
        return _build(_OracleStore, lambda corpus: sparse_mod.BM25Retriever(documents=corpus), OracleEngine())
    finally:
        sparse_mod.B200Engine = saved


def _check_against_nodes(hr, rr, exact_rerank):
    cases = load_golden("reference_nodes")
    assert [c["query"] for c in cases] == QUERIES
    for c in cases:
        q = c["query"]
        # ---- retrieve_node == HybridRetriever.retrieve (nodes.py:51-119)
        got = hr.retrieve(q, top_k=10)
        assert [[d.id, d.text, d.metadata["score"], d.metadata["hybrid_score"]] for d in got] == c["retrieved"]
        assert all(d.text for d in got) and c["retriever_type"] == type(hr).__name__
        assert c["retrieved_count"] == len(got)
        # ---- metadata.user_top_k overrides the node's top_k (nodes.py:64-69); a hybrid top-5 is not a prefix of the
        # top-10: the sub-retrievers get top_k too
        assert [d.id for d in hr.retrieve(q, top_k=5)] == c["top5"]
        # ---- rerank_node == B200Reranker.rerank on the node's prepared copies (nodes.py:138-227)
        rer = rr.rerank(query=q, docs=[Document(id=d.id, text=d.text, metadata=dict(d.metadata)) for d in got], top_k=4)
        if not got:
            assert c["reranked"] == [] and c["reranker_type"] is None
            continue
        assert c["reranker_type"] == type(rr).__name__
        sc = [d.metadata["rerank_score"] for d in rer]
        assert sc == sorted(sc, reverse=True)
        assert all(0.0 <= d.metadata["score"] <= 1.0 and d.metadata["score"] == d.metadata["rerank_score"] for d in rer)
        if exact_rerank:
            assert [[d.id, d.metadata["rerank_score"], d.metadata["score"]] for d in rer] == c["reranked"]
        else:
            # fp16 cross-encoder on the device vs the fp32 host forward of the golden run.  The small random model scores
            # every document of these queries within ~4e-4 of 0.48, inside the 1e-3 cross-encoder tolerance, so which 4
            # documents win and their order are NOT pinned here: this branch checks the plumbing (count, a score within
            # tolerance for every returned document, sorted output).  Cross-encoder accuracy and ranking are tested in
            # tests/test_rerank_gpu.py; retrieval above is compared exactly.
            want = {i: s for i, s, _ in c["reranked"]}
            tol = lambda s: 1e-3 * abs(s) + 1e-4
            assert len(rer) == len(want)
            for pos, d in enumerate(rer):
                if d.id not in want:   # a near tie at the cut-off of the top 4
                    assert abs(d.metadata["rerank_score"] - c["reranked"][pos][1]) <= 2 * tol(c["reranked"][pos][1])
                    continue
                assert abs(d.metadata["rerank_score"] - want[d.id]) <= tol(want[d.id]), (q, d.id)
                gid, gs, _ = c["reranked"][pos]
                assert d.id == gid or abs(want[d.id] - gs) <= 2 * tol(gs)


def test_reference_nodes_drive_the_repo_classes_host_logic(monkeypatch):
    monkeypatch.delenv("BM25_VARIANT", raising=False)
    hr, rr = build_host_stack()
    _check_against_nodes(hr, rr, exact_rerank=True)


@pytest.mark.gpu
def test_reference_nodes_drive_the_repo_classes_on_the_gpu(engine, monkeypatch):
    from sentio_b200.retrievers.sparse import BM25Retriever
    from sentio_b200.vector_store import B200VectorStore

    monkeypatch.delenv("BM25_VARIANT", raising=False)

    def make_store(vecs, ids, payloads):
        st = B200VectorStore(0)
        st.create_collection("Sentio_docs", vecs, ids=ids, payloads=payloads)
        return st

    hr, rr = _build(make_store, lambda corpus: BM25Retriever(documents=corpus), engine)
    _check_against_nodes(hr, rr, exact_rerank=False)


@pytest.mark.gpu
def test_concurrent_retrieve_async_on_one_context(engine, monkeypatch):
    """retrievers/base.py:37-42 dispatches ``retrieve`` to the default thread pool, so one engine context is entered
    from several Python threads at once (ctypes releases the GIL): every call must return exactly the serial answer."""
    import asyncio

    from sentio_b200.retrievers.sparse import BM25Retriever
    from sentio_b200.vector_store import B200VectorStore

    monkeypatch.delenv("BM25_VARIANT", raising=False)

    def make_store(vecs, ids, payloads):
        st = B200VectorStore(0)
        st.create_collection("Sentio_docs", vecs, ids=ids, payloads=payloads)
        return st

    hr, rr = _build(make_store, lambda corpus: BM25Retriever(documents=corpus), engine)
    queries = [f"topic{i % 9} w{i % 13} alpha{i % 5}" for i in range(48)]
    # ids only: like the reference, BM25Retriever hands out the SHARED corpus Documents and the fusion writes
    # metadata["hybrid_score"] into them in place (sparse.py:189-197, hybrid.py:296-297), so under concurrency a document's
    # score field belongs to whichever query wrote last -- the ranking of each call is what must be stable
    serial = [[d.id for d in hr.retrieve(q, top_k=10)] for q in queries]

    async def one(q):
        docs = await hr.retrieve_async(q, top_k=10)
        return [d.id for d in docs]

    async def hammer():
        return await asyncio.gather(*[one(q) for q in queries])

    assert asyncio.run(hammer()) == serial
    # raw threads on the engine itself: dense / BM25 / rerank entry points interleaved on ONE sb_ctx
    emb = HashEmbedder(DIM)
    qv = np.asarray(emb.embed_many_sync(queries), dtype=np.float32)
    st = hr._dense._client  # the B200VectorStore behind the dense retriever
    want = [st.search("Sentio_docs", list(v), limit=7) for v in qv]
    errors, got = [], [None] * len(queries)

    def worker(lo, hi):
        try:
            for i in range(lo, hi):
                got[i] = st.search("Sentio_docs", list(qv[i]), limit=7)
                rr.score_pairs(queries[i], TEXTS[i:i + 3])
        except Exception as exc:  # pragma: no cover
            errors.append(exc)

    threads = [threading.Thread(target=worker, args=(j * 12, (j + 1) * 12)) for j in range(4)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    assert [[(p.id, p.score) for p in r] for r in got] == [[(p.id, p.score) for p in r] for r in want]
