"""Filtered hybrid retrieval (``sb_hybrid_topk_filtered``, ``HybridPipeline.search_hybrid(filters=)``, DESIGN.md K2
"Filtered BM25 and hybrid"): the conditions act on both signals, fusion sees two lists of matching docs only.

* rrf / weighted_rrf / comb_sum against oracle.fusion applied to the filtered dense oracle (oracle.dense over the
  matching rows) and the filtered BM25 oracle (FastBM25 masked, tests/bm25_filter_oracle.py);
* ``filters=None`` is the call without the argument, bit for bit;
* a filtered rerank only ever sees (and returns) matching candidates;
* the partitioned path on one GPU (G in {2, 3} ranks, uneven cuts, shards without a match), with the ``_gather``
  playback of tests/test_sharded_one_gpu.py: bit-identical to one unsharded engine."""
import numpy as np
import pytest

import bm25_filter_oracle as fo

pytestmark = pytest.mark.gpu

N, D, VOCAB = 50_000, 256, 3000
SPLITS = {2: [0, 49_995, 50_000], 3: [0, 6, 23_456, 50_000]}
METHODS = [("rrf", 60, 0.5, 0.5), ("weighted_rrf", 60, 0.7, 0.3), ("comb_sum", 60, 0.7, 0.3)]
# per query: unfiltered, one field, two fields, a code only docs 0..5 hold (one shard at most), -1, a value nobody holds
CONDS = [[], [(0, 2)], [(0, 1), (1, 3)], [(2, 1)], [(1, -1)], [(0, 9)], [(1, 0), (0, 4)], [(2, 0), (0, 3)]]


def _tags():
    d = np.arange(N)
    return {0: (d % 5).astype(np.int32), 1: np.where(d % 13 == 0, -1, (d // 1000) % 4).astype(np.int32),
            2: (d < 6).astype(np.int32)}


@pytest.fixture(scope="module")
def corpus():
    from sentio_b200 import synth
    from sentio_b200.index import build_bm25_from_token_ids

    x = synth.dense_corpus(N, D)
    flat, off = synth.text_corpus_tokens(N, vocab=VOCAB)
    idx = build_bm25_from_token_ids(flat, off, variant="okapi")
    q = synth.query_vectors(len(CONDS), D)
    tok = synth.query_tokens(len(CONDS), vocab=VOCAB)
    terms = [idx.term_ids(t) for t in tok]
    return x, idx, q, terms, _tags()


@pytest.fixture(scope="module")
def single(built_lib, corpus):
    from sentio_b200.engine import B200Engine

    x, idx, _, _, tags = corpus
    e = B200Engine(0)
    e.load_dense(x)
    e.load_bm25(idx)
    for f, c in tags.items():
        e.load_dense_tags(f, c)
        e.load_bm25_tags(f, c)
    yield e
    e.close()


def _bits(a):
    a = np.asarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def _assert_bits(got, want, what):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert np.asarray(g).shape == np.asarray(w).shape and np.array_equal(_bits(g), _bits(w)), what


@pytest.mark.parametrize("method,rrf_k,w_dense,w_sparse", METHODS)
def test_filtered_hybrid_equals_fusion_of_filtered_oracles(single, corpus, method, rrf_k, w_dense, w_sparse):
    from oracle import dense as dense_oracle
    from oracle import fusion as fusion_oracle
    from oracle.rank_bm25_port import FastBM25

    x, idx, q, terms, tags = corpus
    k = 100
    flat, off = single.pack_queries(terms)
    got = single.hybrid_topk(q, flat, off, k, method, rrf_k, w_dense, w_sparse, filters=fo.csr(CONDS))
    fast = FastBM25(idx.indptr, idx.post_doc, idx.post_tf, idx.doc_len, idx.idf, idx.avgdl, "okapi", idx.k1, idx.b,
                    idx.delta)
    for b, conds in enumerate(CONDS):
        m = fo.match_mask(tags, conds, N)
        rows = np.flatnonzero(m)
        dl = []
        if len(rows):
            di, ds = dense_oracle.dense_topk(x[rows], q[b], min(k, len(rows)))
            dl = list(zip(rows[di].tolist(), ds.tolist()))
        s = fast.get_scores(list(terms[b]))
        sl = [(int(i), float(s[i])) for i in fo.filtered_topk(s, m, k)]
        want = fusion_oracle.fuse(method, rrf_k, w_dense, w_sparse, dl, sl, [], k)
        n = int(got[3][b])
        assert n == len(want), (method, b)
        assert got[0][b, :n].tolist() == [w[0] for w in want], (method, b)
        assert got[1][b, :n].tolist() == [w[1] for w in want], (method, b)
        assert m[got[0][b, :n]].all()
    assert got[3][4] == 0 and got[3][5] == 0 and 0 < got[3][3] <= 6


def test_filters_none_is_the_call_without_it(single, corpus):
    from sentio_b200.pipeline import HybridPipeline

    _, _, q, terms, _ = corpus
    flat, off = single.pack_queries(terms)
    _assert_bits(single.hybrid_topk(q, flat, off, 100, filters=None), single.hybrid_topk(q, flat, off, 100), "engine")
    _assert_bits(single.bm25_topk(terms, 100, filters=None), single.bm25_topk(terms, 100), "bm25")
    p = HybridPipeline(0, engine=single)
    _assert_bits(p.search_hybrid(q, terms, 100, filters=None), p.search_hybrid(q, terms, 100), "pipeline")
    _assert_bits(p.search_dense(q, 100, filters=None), p.search_dense(q, 100), "dense")
    # conditions that name no query: exactly the unfiltered path
    _assert_bits(p.search_hybrid(q, terms, 100, filters=fo.csr([[]] * len(CONDS))), p.search_hybrid(q, terms, 100),
                 "empty CSR")


def test_pipeline_single_shard_equals_engine(single, corpus):
    from sentio_b200.pipeline import HybridPipeline

    _, _, q, terms, _ = corpus
    flat, off = single.pack_queries(terms)
    p = HybridPipeline(0, engine=single)
    for method, rrf_k, wd, ws in METHODS:
        _assert_bits(p.search_hybrid(q, terms, 100, method, rrf_k, wd, ws, filters=fo.csr(CONDS)),
                     single.hybrid_topk(q, flat, off, 100, method, rrf_k, wd, ws, filters=fo.csr(CONDS)), method)


def test_hybrid_errors(single, corpus):
    from sentio_b200._lib import SentioB200ArgError, SentioB200Error

    _, _, q, terms, _ = corpus
    flat, off = single.pack_queries(terms[:1])
    with pytest.raises(SentioB200ArgError):
        single.hybrid_topk(q[:1], flat, off, 10, filters=fo.csr([[(16, 0)]]))
    with pytest.raises(SentioB200Error):
        single.hybrid_topk(q[:1], flat, off, 10, filters=fo.csr([[(7, 0)]]))     # loaded in neither index


def test_filtered_rerank_sees_only_matching_candidates(built_lib, corpus):
    from sentio_b200.cross_encoder import CrossEncoderWeights
    from sentio_b200.pipeline import HybridPipeline

    x, idx, q, terms, tags = corpus
    p = HybridPipeline(0)
    try:
        p.load_dense(x)
        p.load_bm25(idx)
        for f, c in tags.items():
            p.load_tags(f, c)
        p.load_cross_encoder(CrossEncoderWeights.random_minilm_l6(seed=3))
        rng = np.random.default_rng(9)
        ld = 24
        p.load_doc_tokens(rng.integers(1000, 30000, (N, ld)).astype(np.uint16), rng.integers(4, ld + 1, N).astype(np.int32))
        q_tok = rng.integers(1000, 30000, (len(CONDS), 8)).astype(np.int32)
        q_len = np.full(len(CONDS), 8, np.int32)
        ids, sc, cnt = p.search_hybrid_rerank(q, terms, q_tok, q_len, 50, 10, seq_len=64, filters=fo.csr(CONDS))
        fused = p.search_hybrid(q, terms, 50, filters=fo.csr(CONDS))
        for b, conds in enumerate(CONDS):
            m = fo.match_mask(tags, conds, N)
            n = int(cnt[b])
            assert n == min(10, int(fused[3][b])), b
            assert m[ids[b, :n]].all(), b
            assert set(ids[b, :n].tolist()) <= set(fused[0][b, :int(fused[3][b])].tolist()), b
    finally:
        p.engine.close()


def _sharded_pipeline_class():
    from sentio_b200.pipeline import HybridPipeline

    class OneGpuShard(HybridPipeline):
        """HybridPipeline whose all-gather is played back from records harvested in a first pass."""

        def __init__(self, rank, world, box):
            super().__init__(0, rank=rank, world=world)
            self.box = box

        def _gather(self, rec):
            t = self.torch
            if self.box["mode"] == "harvest":
                self.box["recs"][self.rank] = rec.clone()
                return t.zeros((self.world, rec.numel()), dtype=t.uint8, device=rec.device)
            return t.stack(self.box["recs"])

    return OneGpuShard


@pytest.fixture(scope="module", params=[2, 3])
def ranks(request, built_lib, corpus):
    G = request.param
    x, idx, _, _, tags = corpus
    box = {"mode": "harvest", "recs": [None] * G}
    cls = _sharded_pipeline_class()
    pipes = [cls(r, G, box) for r in range(G)]
    cuts = SPLITS[G]
    for r, p in enumerate(pipes):
        p.load_dense(x[cuts[r]:cuts[r + 1]], id_base=cuts[r])
        p.load_bm25(idx.shard(cuts[r], cuts[r + 1]), id_base=cuts[r])
        for f, c in tags.items():
            p.load_tags(f, c)          # the corpus-global column: each rank keeps its own slice
    yield G, pipes, box
    for p in pipes:
        p.engine.close()


def _two_pass(pipes, box, call):
    box["mode"] = "harvest"
    for p in pipes:
        call(p)
    box["mode"] = "replay"
    return [call(p) for p in pipes]


@pytest.mark.parametrize("k", [10, 100])
def test_sharded_filtered_dense_equals_single_engine(ranks, single, corpus, k):
    G, pipes, box = ranks
    _, _, q, _, _ = corpus
    want = single.dense_topk(q, k, filters=fo.csr(CONDS))
    for r, got in enumerate(_two_pass(pipes, box, lambda p: p.search_dense(q, k, filters=fo.csr(CONDS)))):
        _assert_bits(got, want, (G, k, r))


@pytest.mark.parametrize("method,rrf_k,w_dense,w_sparse", METHODS)
@pytest.mark.parametrize("k", [10, 100])
def test_sharded_filtered_hybrid_equals_single_engine(ranks, single, corpus, method, rrf_k, w_dense, w_sparse, k):
    G, pipes, box = ranks
    _, _, q, terms, _ = corpus
    flat, off = single.pack_queries(terms)
    want = single.hybrid_topk(q, flat, off, k, method, rrf_k, w_dense, w_sparse, filters=fo.csr(CONDS))
    got_all = _two_pass(pipes, box, lambda p: p.search_hybrid(q, terms, k, method, rrf_k, w_dense, w_sparse,
                                                              filters=fo.csr(CONDS)))
    for r, got in enumerate(got_all):
        _assert_bits(got, want, (G, method, k, r))
