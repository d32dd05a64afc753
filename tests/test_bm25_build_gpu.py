"""§8f row 2: the sort-based GPU index build (sb_bm25_build_*) produces exactly the index the host builder
(sentio_b200/index.py, itself pinned to rank_bm25's state by tests/test_oracle_golden.py) produces: same term ids
(first-occurrence order), same CSR, same df / idf / avgdl bit for bit, and therefore bit-identical scores."""
import numpy as np
import pytest

from conftest import load_golden
from sentio_b200 import synth
from sentio_b200.index import build_bm25_from_texts, build_bm25_from_token_ids, tokenize_texts

pytestmark = pytest.mark.gpu


def _assert_same_index(got, want):
    assert got.n_docs == want.n_docs and got.avgdl == want.avgdl and got.average_idf == want.average_idf
    assert np.array_equal(got.idf, want.idf)
    assert np.array_equal(got.indptr, want.indptr)
    assert np.array_equal(got.post_doc, want.post_doc)
    assert np.array_equal(got.post_tf, want.post_tf)
    assert np.array_equal(got.doc_len, want.doc_len)
    n = min(len(got.token_id_map), len(want.token_id_map))
    assert np.array_equal(got.token_id_map[:n], want.token_id_map[:n])
    assert np.all(got.token_id_map[n:] == -1) and np.all(want.token_id_map[n:] == -1)


@pytest.mark.parametrize("variant,n,vocab", [("okapi", 30000, 5000), ("plus", 7000, 800), ("okapi", 33, 12)])
def test_gpu_build_equals_host_build(engine, variant, n, vocab):
    flat, off = synth.text_corpus_tokens(n, vocab=vocab)
    flat = (flat * 7 + 3).astype(np.int32)  # sparse raw ids, not in first-occurrence order
    want = build_bm25_from_token_ids(flat, off, variant=variant)
    got = engine.build_bm25_gpu(flat, off, variant=variant, export=True)
    _assert_same_index(got, want)
    # the installed device index scores exactly like the uploaded host index
    queries = (synth.query_tokens(20, vocab=vocab) * 7 + 3).astype(np.int32)
    terms = [got.term_ids(q) for q in queries] + [np.array([-1], np.int32)]
    a = engine.bm25_topk(terms, 50)
    sc_a = [engine.bm25_scores(t) for t in terms[:3]]
    engine.load_bm25(want)
    b = engine.bm25_topk([want.term_ids(q) for q in queries] + [np.array([-1], np.int32)], 50)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    for t, s in zip(terms[:3], sc_a):
        assert np.array_equal(engine.bm25_scores(t), s)


def _edge_stream(kind):
    if kind == "empty_docs":     # zero-length docs first, last and in runs between non-empty ones
        lens = np.array([0, 3, 0, 0, 5, 1, 0, 2, 0])
        flat = np.arange(lens.sum()) % 4 + 10
    elif kind == "tf_max":       # one term 65535 times in a doc (the uint16 limit), next to ordinary docs
        lens = np.array([2, 65535, 3, 65536])
        flat = np.concatenate([[1, 2], np.full(65535, 7), [7, 1, 3], np.full(65535, 1), [7]])
    else:                        # a single doc
        lens = np.array([4])
        flat = np.array([9, 4, 9, 9])
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    return flat.astype(np.int32), off


@pytest.mark.parametrize("kind", ["empty_docs", "tf_max", "one_doc"])
@pytest.mark.parametrize("variant", ["okapi", "plus"])
def test_gpu_build_equals_host_build_at_the_edges(engine, kind, variant):
    flat, off = _edge_stream(kind)
    want = build_bm25_from_token_ids(flat, off, variant=variant)
    got = engine.build_bm25_gpu(flat, off, variant=variant, export=True)
    _assert_same_index(got, want)
    if kind == "tf_max":
        assert want.post_tf.max() == 65535
    terms = [got.term_ids(q) for q in ([7], [1, 7, 3], [9, 4, 9], [10, 11, 12, 13], [2, 99])]
    a = engine.bm25_topk(terms, 8)
    sc_a = [engine.bm25_scores(t) for t in terms]
    engine.load_bm25(want)
    b = engine.bm25_topk(terms, 8)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint64) if x.dtype == np.float64 else x,
                              y.view(np.uint64) if y.dtype == np.float64 else y)
    for t, s in zip(terms, sc_a):
        assert np.array_equal(engine.bm25_scores(t).view(np.uint64), s.view(np.uint64))


def test_gpu_build_without_export_keeps_postings_on_device(engine):
    flat, off = synth.text_corpus_tokens(5000, vocab=700)
    want = build_bm25_from_token_ids(flat, off)
    got = engine.build_bm25_gpu(flat, off)
    assert len(got.post_doc) == 0 and got.extras["postings_on_host"] is False
    assert np.array_equal(got.idf, want.idf)
    q = synth.query_tokens(8, vocab=700)
    a = engine.bm25_topk([got.term_ids(t) for t in q], 10)
    engine.load_bm25(want)
    b = engine.bm25_topk([want.term_ids(t) for t in q], 10)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("variant", ["okapi", "plus"])
def test_gpu_build_on_golden_text_corpora(engine, variant):
    for c in [x for x in load_golden("bm25") if x["variant"] == variant]:
        want = build_bm25_from_texts(c["texts"], variant=variant)
        vocab, flat, off = tokenize_texts(c["texts"])
        got = engine.build_bm25_gpu(flat, off, variant=variant, export=True)
        assert np.array_equal(got.idf, want.idf) and np.array_equal(got.indptr, want.indptr)
        assert np.array_equal(got.post_doc, want.post_doc) and np.array_equal(got.post_tf, want.post_tf)
        for qc in c["queries"]:
            terms = np.asarray([vocab.get(t, -1) for t in qc["query"].lower().split()], np.int32)
            assert np.array_equal(engine.bm25_scores(terms), np.asarray(qc["scores"]))


def test_gpu_build_rejects_bad_streams(engine):
    from sentio_b200._lib import SentioB200Error

    with pytest.raises(SentioB200Error):
        engine.build_bm25_gpu(np.array([1, -2, 3], np.int32), np.array([0, 3], np.int64))
    with pytest.raises(SentioB200Error):  # tf above uint16
        engine.build_bm25_gpu(np.zeros(70000, np.int32), np.array([0, 70000], np.int64))


def test_full_size_1m_docs_gpu_build(engine):
    """BASELINE config 3 corpus (1 M docs, ~80 M tokens): device build == host build (df, idf, CSR) and it is fast."""
    import time

    flat, off = synth.text_corpus_tokens(1_000_000)
    t0 = time.perf_counter()
    got = engine.build_bm25_gpu(flat, off, export=True)
    gpu_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    want = build_bm25_from_token_ids(flat, off)
    cpu_s = time.perf_counter() - t0
    print(f"BM25 index build, 1 M docs / {len(flat)} tokens: GPU {gpu_s:.2f} s (incl. H2D + export), host NumPy {cpu_s:.2f} s")
    _assert_same_index(got, want)
