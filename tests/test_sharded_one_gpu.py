"""The sharded hybrid path on one GPU: G in {2, 3, 4} HybridPipeline ranks, each with its own B200Engine on device 0,
over a corpus cut at uneven split points (one shard holds fewer rows than k).  A test subclass replaces only
``_gather`` (the NCCL all-gather) and runs every call twice:

  pass 1: ``_gather`` keeps a copy of the rank's packed record and returns an all-zero buffer (counts 0 -> empty merge);
  pass 2: ``_gather`` returns the G harvested records stacked, exactly what all_gather_into_tensor would deliver.

Everything else is the product code (record packing, K6 merge_shards_dev, K3 fuse_dev), and every rank's
``search_dense`` / ``search_hybrid`` must be BIT-IDENTICAL to one unsharded engine's ``dense_topk`` / ``hybrid_topk``
(the sb_hybrid_topk host entry, a separate code path).  Ties across shards: duplicate dense rows in different shards, the
BM25Plus variant (every doc scores > 0, docs without a query term tie massively), a zero query vector, an empty and an
unknown-only term list.  A few queries are also checked against oracle.dense + FastBM25 + oracle.fusion.
(The multi-process NCCL path itself is exercised by scripts/check_multigpu.py.)"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, D, VOCAB = 50_000, 256, 3000
SPLITS = {2: [0, 49_995, 50_000], 3: [0, 6, 23_456, 50_000], 4: [0, 17_000, 17_003, 31_111, 50_000]}
DUP_PAIRS = [(100, 49_997), (3, 40_000), (17_001, 20_000), (30_000, 31_500)]   # (source row, copy) in other shards
METHODS = [("rrf", 60, 0.5, 0.5), ("weighted_rrf", 60, 0.7, 0.3), ("comb_sum", 60, 0.7, 0.3)]


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


@pytest.fixture(scope="module")
def corpus():
    from sentio_b200 import synth
    from sentio_b200.index import build_bm25_from_token_ids

    x = synth.dense_corpus(N, D)
    for src, dst in DUP_PAIRS:
        x[dst] = x[src]
    flat, off = synth.text_corpus_tokens(N, vocab=VOCAB)
    idx = {v: build_bm25_from_token_ids(flat, off, variant=v) for v in ("okapi", "plus")}
    q = synth.query_vectors(12, D)
    q = np.concatenate([q, x[[s for s, _ in DUP_PAIRS]].astype(np.float32), np.zeros((1, D), np.float32)])
    tok = synth.query_tokens(len(q), vocab=VOCAB)
    terms = {v: [idx[v].term_ids(t) for t in tok] for v in idx}
    for v in terms:
        terms[v][2] = np.zeros(0, np.int32)                          # a query without text
        terms[v][3] = idx[v].term_ids([VOCAB + 5, 10 ** 7])          # only unknown tokens
        assert (terms[v][3] == -1).all()
    return x, idx, q, terms


@pytest.fixture(scope="module")
def single(built_lib, corpus):
    from sentio_b200.engine import B200Engine

    x, idx, _, _ = corpus
    e = B200Engine(0)
    e.load_dense(x)
    yield e
    e.close()


@pytest.fixture(scope="module", params=[2, 3, 4])
def ranks(request, built_lib, corpus):
    G = request.param
    x, _, _, _ = corpus
    box = {"mode": "harvest", "recs": [None] * G}
    cls = _sharded_pipeline_class()
    pipes = [cls(r, G, box) for r in range(G)]
    cuts = SPLITS[G]
    for r, p in enumerate(pipes):
        p.load_dense(x[cuts[r]:cuts[r + 1]], id_base=cuts[r])
    yield G, pipes, box
    for p in pipes:
        p.engine.close()


def _load_bm25(single, pipes, idx, G):
    """The whole index on the single engine, shard r's postings (global idf / avgdl) on rank r."""
    cuts = SPLITS[G]
    if single.bm25 is not idx:
        single.load_bm25(idx)
    for r, p in enumerate(pipes):
        if p.engine.bm25 is None or p.engine.bm25.extras.get("whole") is not idx:
            sh = idx.shard(cuts[r], cuts[r + 1])
            sh.extras["whole"] = idx
            p.load_bm25(sh, id_base=cuts[r])


def _two_pass(pipes, box, call):
    box["mode"] = "harvest"
    for p in pipes:
        call(p)
    box["mode"] = "replay"
    return [call(p) for p in pipes]


def _assert_bits(got, want, what):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        g, w = np.asarray(g), np.asarray(w)
        assert g.dtype == w.dtype and g.shape == w.shape, what
        if g.dtype == np.float64:
            g, w = g.view(np.uint64), w.view(np.uint64)
        assert np.array_equal(g, w), what


@pytest.mark.parametrize("k", [10, 100, 1024])
def test_sharded_dense_equals_single_engine(ranks, single, corpus, k):
    G, pipes, box = ranks
    _, _, q, _ = corpus
    want = single.dense_topk(q, k)
    for r, got in enumerate(_two_pass(pipes, box, lambda p: p.search_dense(q, k))):
        _assert_bits(got, want, (G, k, r))
    # duplicate rows in different shards tie at the top: the lower id comes first
    for b, (src, dst) in enumerate(DUP_PAIRS):
        row = 12 + b
        assert want[0][row, :2].tolist() == [src, dst] and want[1][row, 0] == want[1][row, 1]


@pytest.mark.parametrize("variant", ["okapi", "plus"])
@pytest.mark.parametrize("method,rrf_k,w_dense,w_sparse", METHODS)
@pytest.mark.parametrize("k", [10, 100, 1024])
def test_sharded_hybrid_equals_single_engine(ranks, single, corpus, variant, method, rrf_k, w_dense, w_sparse, k):
    G, pipes, box = ranks
    _, idx, q, terms = corpus
    _load_bm25(single, pipes, idx[variant], G)
    flat, off = single.pack_queries(terms[variant])
    want = single.hybrid_topk(q, flat, off, k, method, rrf_k, w_dense, w_sparse)
    got_all = _two_pass(pipes, box, lambda p: p.search_hybrid(q, terms[variant], k, method, rrf_k, w_dense, w_sparse))
    for r, got in enumerate(got_all):
        _assert_bits(got, want, (G, variant, method, k, r))
    if variant == "plus":
        # every doc scores > 0: the sparse list of a normal query is full, so the fused list is too
        assert (want[3][[0, 1]] == k).all()


@pytest.mark.parametrize("variant", ["okapi", "plus"])
@pytest.mark.parametrize("method,rrf_k,w_dense,w_sparse", METHODS)
def test_sharded_hybrid_equals_oracle_on_a_few_queries(ranks, single, corpus, variant, method, rrf_k, w_dense,
                                                       w_sparse):
    from oracle import dense as dense_oracle
    from oracle import fusion as fusion_oracle
    from oracle.rank_bm25_port import FastBM25

    G, pipes, box = ranks
    if G != 3:
        pytest.skip("one shard count is enough for the oracle check")
    x, idx, q, terms = corpus
    ix = idx[variant]
    _load_bm25(single, pipes, ix, G)
    k = 100
    got = _two_pass(pipes, box, lambda p: p.search_hybrid(q, terms[variant], k, method, rrf_k, w_dense, w_sparse))[1]
    fast = FastBM25(ix.indptr, ix.post_doc, ix.post_tf, ix.doc_len, ix.idf, ix.avgdl, variant, ix.k1, ix.b, ix.delta)
    for b in (0, 1, 2, 3, 12):
        di, ds = dense_oracle.dense_topk(x, q[b], k)
        s = fast.get_scores([t for t in terms[variant][b]])
        order = [i for i in np.argsort(-s, kind="stable")[:k] if s[i] > 0]
        want = fusion_oracle.fuse(method, rrf_k, w_dense, w_sparse, list(zip(di.tolist(), ds.tolist())),
                                  [(int(i), float(s[i])) for i in order], [], k)
        n = int(got[3][b])
        assert n == len(want), (variant, method, b)
        assert got[0][b, :n].tolist() == [w[0] for w in want], (variant, method, b)
        assert got[1][b, :n].tolist() == [w[1] for w in want], (variant, method, b)
