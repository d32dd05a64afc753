"""K2 (BM25) at its edges: ``sb_bm25_scores`` bit-identical to FastBM25 and ``bm25_topk`` identical to the rank_bm25
order (ids, score bits, counts, -1 / 0.0 padding) at the range, strip, sub-batch, head-term, query-length, top-k and
score edges.  Inputs and references: tests/bm25_edges.py; tests/test_bm25_edges_cpu.py shows they can see seeded defects."""
import numpy as np
import pytest

import bm25_edges as be
from sentio_b200.document import Document

pytestmark = pytest.mark.gpu

VARIANTS = ["okapi", "plus"]


def _device():
    import torch

    return torch.cuda.get_device_properties(0)


def _check(engine, case, scores_rows=(), rows=None, dev=False):
    """Loads the case, compares the top-k of `rows` (default: case.rows or all) and the full scores of `scores_rows`."""
    engine.load_bm25(case.idx, id_base=case.id_base)
    f = be.fast(case.idx)
    ids, sc, cnt = engine.bm25_topk(case.queries, case.k)
    rows = (case.rows if case.rows is not None else range(len(case.queries))) if rows is None else rows
    for b in rows:
        s = f.get_scores(list(case.queries[b]))
        o = be.ref_topk(s, case.k)
        w_ids, w_sc, w_cnt = be.padded([o], [s], case.k, case.id_base)
        assert int(cnt[b]) == int(w_cnt[0]), (case.name, b)
        assert np.array_equal(ids[b], w_ids[0]), (case.name, b)
        assert np.array_equal(be.bits(sc[b]), be.bits(w_sc[0])), (case.name, b)
    for b in scores_rows:
        want = f.get_scores(list(case.queries[b]))
        assert np.array_equal(be.bits(engine.bm25_scores(case.queries[b])), be.bits(want)), (case.name, b)
    if dev:
        import torch

        flat, off = engine.pack_queries(case.queries)
        d = engine.bm25_topk_dev(torch.from_numpy(flat).cuda(), torch.from_numpy(off).cuda(), len(case.queries),
                                 int(off[-1]), int(np.diff(off).max()), case.k)
        torch.cuda.synchronize()
        for a, x in zip((ids, sc, cnt), d):
            x = x.cpu().numpy()
            assert np.array_equal(a.view(np.uint64) if a.dtype == np.float64 else a,
                                  x.view(np.uint64) if x.dtype == np.float64 else x), case.name
    return ids, sc, cnt


@pytest.mark.parametrize("n", [1, 31, 33, 511, 512, 513, 4095, 4096, 4097, 8191, 8192, 8193, 3 * 8192 + 1, 4 * 8192 + 1,
                               5 * 8192 - 1])
@pytest.mark.parametrize("variant", VARIANTS)
def test_postings_at_range_and_sub_range_edges(engine, n, variant):
    case = be.range_edge_case(n, variant)
    _check(engine, case, scores_rows=range(len(case.queries)))


@pytest.mark.parametrize("variant", VARIANTS)
def test_strips_and_sub_batches(engine, variant):
    case = be.strip_case(variant)
    n, B = case.idx.n_docs, len(case.queries)
    sbq = be.sub_batch_size(n, B)
    sms = _device().multi_processor_count
    assert sbq < B
    for b0 in range(0, B, sbq):
        assert be.ranges_per_cta(sms, min(sbq, B - b0), n) > 1, (b0, sms)
    _check(engine, case, scores_rows=[0, B - 1], dev=True)


@pytest.mark.parametrize("n", [4095, 4096, 4097, 8193])
@pytest.mark.parametrize("variant", VARIANTS)
def test_head_terms_at_the_dense_row_edges(engine, monkeypatch, n, variant):
    case = be.head_case(n, variant)
    df = np.diff(case.idx.indptr)
    t1, t2 = case.idx.term_ids([1, 2])
    assert df[t1] * 4 >= n and (n % 4 or df[t1] * 4 == n) and (n % 4 != 1 or df[t2] * 4 == n - 1)
    got = _check(engine, case, scores_rows=range(len(case.queries)))
    monkeypatch.setenv("SB_BM25_DENSE", "0")
    _check_same_without_dense_rows(engine, case, got)


def _check_same_without_dense_rows(engine, case, got):
    engine.load_bm25(case.idx, id_base=case.id_base)
    again = engine.bm25_topk(case.queries, case.k)
    for a, b in zip(got, again):
        assert np.array_equal(a.view(np.uint64) if a.dtype == np.float64 else a,
                              b.view(np.uint64) if b.dtype == np.float64 else b), case.name
    f = be.fast(case.idx)
    for t in case.queries[:3]:
        assert np.array_equal(be.bits(engine.bm25_scores(t)), be.bits(f.get_scores(list(t))))


@pytest.mark.parametrize("variant", VARIANTS)
def test_more_head_terms_than_dense_rows(engine, monkeypatch, variant):
    case = be.many_heads_case(variant)
    heads = be.head_terms(case.idx)
    assert len(heads) == 70 > be.MAX_ROWS
    got = _check(engine, case, scores_rows=range(len(case.queries)))
    monkeypatch.setenv("SB_BM25_DENSE", "0")
    _check_same_without_dense_rows(engine, case, got)


@pytest.mark.parametrize("variant", VARIANTS)
def test_queries_of_any_length(engine, variant):
    case = be.long_query_case(variant)
    lens = [len(q) for q in case.queries]
    assert max(lens) > be.max_term_block(_device().shared_memory_per_block_optin)
    _check(engine, case, scores_rows=range(len(case.queries)), dev=True)
    # one long query among short ones, in a batch of its own
    one = be.Case(case.name + "_one", case.idx, [case.queries[i] for i in (0, 3, 9, 1, 2)], k=case.k)
    _check(engine, one)


@pytest.mark.parametrize("variant", VARIANTS)
def test_retriever_with_a_5000_token_query(monkeypatch, variant):
    monkeypatch.delenv("BM25_VARIANT", raising=False)
    from sentio_b200.retrievers.sparse import BM25Retriever

    rng = np.random.default_rng(21)
    texts = [" ".join(f"w{rng.integers(0, 400)}" for _ in range(rng.integers(3, 30))) for _ in range(2000)]
    r = BM25Retriever(documents=[Document(id=f"d{i}", text=t) for i, t in enumerate(texts)], variant=variant)
    long_q = " ".join(f"w{x}" for x in rng.integers(0, 450, 5000))
    f = be.fast(r.bm25)
    want = f.get_scores(list(r.bm25.term_ids(long_q.split())))
    order = be.ref_topk(want, 50)
    assert len(order) == 50
    got = r.retrieve(long_q, top_k=50)
    assert [d.id for d in got] == [f"d{i}" for i in order]
    assert [d.metadata["bm25_score"] for d in got] == [float(want[i]) for i in order]
    batch = r.retrieve_batch(["w1 w2", long_q, "w3"], top_k=50)
    assert [d.id for d in batch[1]] == [f"d{i}" for i in order]
    assert [d.metadata["bm25_score"] for d in batch[1]] == [float(want[i]) for i in order]
    assert len(batch[0]) > 0 and len(batch[2]) > 0


@pytest.mark.parametrize("k", [1, 32, 33, 1000, 1024])
@pytest.mark.parametrize("variant", VARIANTS)
def test_top_k_sizes(engine, k, variant):
    case = be.k_sweep_case(variant, k)
    ids, sc, cnt = _check(engine, case)
    if variant == "okapi":
        assert int(cnt[-2]) == 4 < k or k < 4     # k above the number of positive docs: -1 / 0.0 padding
        assert (ids[-2, cnt[-2]:] == -1).all() and (be.bits(sc[-2, cnt[-2]:]) == 0).all()


@pytest.mark.parametrize("m", [12287, 12288, 12289, 40000])
@pytest.mark.parametrize("variant", VARIANTS)
def test_all_tie_corpus(engine, m, variant):
    case = be.tie_case(m, variant)
    if variant == "okapi":
        s = be.fast(case.idx).get_scores(list(case.queries[0]))
        assert len(be.candidates(s, case.k)) == m
    _check(engine, case)


@pytest.mark.parametrize("variant", VARIANTS)
def test_winners_at_both_ends_of_more_candidates_than_the_stage(engine, variant):
    case = be.both_ends_case(variant)
    s = be.fast(case.idx).get_scores(list(case.queries[0]))
    assert len(be.candidates(s, case.k)) > be.STAGE
    _check(engine, case)


@pytest.mark.parametrize("variant", VARIANTS)
def test_ties_straddling_rank_k_with_a_large_id_base(engine, variant):
    case = be.straddle_case(variant)
    s = be.fast(case.idx).get_scores(list(case.queries[0]))
    o = be.ref_topk(s, case.k + 200)
    assert s[o[case.k - 1]] == s[o[case.k]]              # rank k splits a tie group ...
    tie = np.flatnonzero(s == s[o[case.k - 1]])
    assert len(np.unique(tie // be.RANGE)) == 5                 # ... spread over all five ranges
    ids, _, cnt = _check(engine, case)
    assert (ids[0, :cnt[0]] >= 1 << 40).all()


@pytest.mark.parametrize("kind", ["empty_sampled", "exact_ks", "tight"])
def test_sample_bound_edges(engine, kind):
    case = be.sample_case(kind)
    s = be.fast(case.idx).get_scores(list(case.queries[0]))
    if kind == "tight":
        assert len(be.candidates(s, case.k)) == 12 and len(be.candidates(s, case.k, floor=True)) == 8
    else:
        assert (be.ref_topk(s, case.k) >= 4 * be.RANGE).all()
    for k in (1, 3, 10, 12, 13, 100):
        _check(engine, be.Case(case.name, case.idx, case.queries, k=k), scores_rows=[0])


@pytest.mark.parametrize("kind,variant", [("idf_zero", "okapi"), ("negative_floor", "okapi"), ("empty_docs", "okapi"),
                                          ("empty_docs", "plus"), ("tf_max", "okapi"), ("tf_max", "plus"),
                                          ("k1_0", "okapi"), ("k1_0", "plus"), ("b_0", "okapi"), ("b_0", "plus"),
                                          ("b_1", "okapi"), ("b_1", "plus")])
def test_score_extremes(engine, kind, variant):
    case = be.extreme_case(kind, variant)
    idx = case.idx
    if kind == "idf_zero":
        assert idx.idf[idx.term_ids([1])[0]] == 0.0
    elif kind == "negative_floor":
        assert idx.average_idf < 0 and idx.idf[idx.term_ids([1])[0]] < 0
    elif kind == "empty_docs":
        assert (idx.doc_len == 0).sum() > 1000
    elif kind == "tf_max":
        assert idx.post_tf.max() == 65535
    ids, sc, cnt = _check(engine, case, scores_rows=range(len(case.queries)))
    if kind == "negative_floor":
        assert int(cnt[1]) == 0 and (ids[1] == -1).all()
