"""Filtered BM25 (``sb_bm25_topk_filtered[_dev]``, DESIGN.md K2 "Filtered BM25 and hybrid") against FastBM25 scores
masked by the conditions and cut with the unfiltered rule (tests/bm25_filter_oracle.py): ids, score bits, counts and
the -1 / 0.0 padding must match exactly.  Two cases are built to see a filter ignored by one of the two passes:

* ``test_low_scoring_matches_behind_high_scoring_non_matches``: every high-scoring doc fails the filter and the matching
  docs score low.  A sample pass that ignored the filter would set the collect threshold among the high scores and no
  match would survive; a collect pass that ignored the filter would return the high-scoring non-matching docs."""
import numpy as np
import pytest

import bm25_edges as be
import bm25_filter_oracle as fo

pytestmark = pytest.mark.gpu

VARIANTS = ["okapi", "plus"]
N_A = 5 * be.RANGE - 1000   # 5 ranges: the sample ranges are 0..3, range 4 is never sampled


def _tags_a(n):
    d = np.arange(n)
    return {0: (d % 7).astype(np.int32), 1: ((d // 3) % 5).astype(np.int32), 2: (d // be.RANGE).astype(np.int32),
            3: np.where(d % 11 == 0, -1, d % 2).astype(np.int32), 5: np.zeros(n, np.int32)}


def _load(engine, idx, tags, id_base=0):
    engine.load_bm25(idx, id_base=id_base)
    for f, c in tags.items():
        engine.load_bm25_tags(f, c)


def _check(engine, idx, queries, conds, k, tags, id_base=0, rows=None):
    """engine's filtered top-k of every query against the reference; unfiltered rows against bm25_topk bit for bit."""
    f = be.fast(idx)
    n = idx.n_docs
    got = engine.bm25_topk(queries, k, filters=fo.csr(conds))
    plain = engine.bm25_topk(queries, k)
    for b in (range(len(queries)) if rows is None else rows):
        s = f.get_scores(list(queries[b]))
        o = fo.filtered_topk(s, fo.match_mask(tags, conds[b], n), k)
        w = fo.padded([o], [s], k, id_base)
        assert int(got[2][b]) == int(w[2][0]), (b, conds[b])
        assert np.array_equal(got[0][b], w[0][0]), (b, conds[b])
        assert np.array_equal(be.bits(got[1][b]), be.bits(w[1][0])), (b, conds[b])
        if not conds[b]:
            for g, p in zip(got, plain):
                assert np.array_equal(be.bits(g[b]) if g.dtype == np.float64 else g[b],
                                      be.bits(p[b]) if p.dtype == np.float64 else p[b]), b
    return got


def _corpus_a(variant):
    rng = np.random.default_rng(3)
    n = N_A
    d = np.repeat(np.arange(n), 3)
    t = rng.integers(0, 500, len(d))
    idx = be.index_from_triples(n, d, t, 1, fill=1 + np.arange(n) % 4, variant=variant)
    queries = [idx.term_ids(list(rng.integers(0, 500, 4))) for _ in range(6)] + [idx.term_ids([3, be.UNKNOWN])]
    return idx, queries


CONDS_A = [[], [(0, 3)], [(0, 3), (1, 2)], [(0, 3), (1, 2), (3, 1)], [(0, -1)], [(2, 4)], [(2, 1)], [(3, 0)], [(5, 0)],
           [(1, 4), (1, 4)], [(0, 9)]]


@pytest.mark.parametrize("k", [1, 100, 1024])
@pytest.mark.parametrize("variant", VARIANTS)
def test_conditions_on_one_to_three_fields_mixed_with_unfiltered(engine, variant, k):
    """1-3 fields, an unknown value (-1) and a value no doc holds, matches only in the never-sampled range 4 ((2, 4)) and
    only in sample range 1 ((2, 1)), unfiltered queries in the same batch."""
    idx, qs = _corpus_a(variant)
    tags = _tags_a(idx.n_docs)
    _load(engine, idx, tags, id_base=1000)
    queries = [qs[i % len(qs)] for i in range(len(CONDS_A))]
    got = _check(engine, idx, queries, CONDS_A, k, tags, id_base=1000)
    assert got[2][4] == 0 and got[2][10] == 0   # code -1 and an absent value return nothing
    assert (got[0][5][:got[2][5]] >= 1000 + 4 * be.RANGE).all() and got[2][5] > 0
    assert got[2][0] > 0


@pytest.mark.parametrize("variant", VARIANTS)
def test_filter_matching_everything_is_the_unfiltered_call(engine, variant):
    idx, qs = _corpus_a(variant)
    tags = _tags_a(idx.n_docs)
    _load(engine, idx, tags)
    for k in (1, 100, 1024):
        got = engine.bm25_topk(qs, k, filters=fo.csr([[(5, 0)]] * len(qs)))
        want = engine.bm25_topk(qs, k)
        for g, w in zip(got, want):
            assert np.array_equal(be.bits(g) if g.dtype == np.float64 else g, be.bits(w) if w.dtype == np.float64 else w)


@pytest.mark.parametrize("variant", VARIANTS)
def test_match_set_sizes(engine, variant):
    """Matching sets of size 0, 1, exactly k, fewer than k positive matches, and a set whose docs hold no query term
    (nothing under Okapi; under Plus every one of them at the sum of idf * delta)."""
    n, k = 3 * be.RANGE + 17, 100
    rng = np.random.default_rng(5)
    holders = np.sort(rng.choice(n, 4000, replace=False))            # docs holding term 1
    idx = be.index_from_triples(n, holders, np.full(len(holders), 1), 1 + holders % 3, fill=1 + np.arange(n) % 5,
                                variant=variant)
    others = np.setdiff1d(np.arange(n), holders)
    col = np.full(n, -1, np.int32)
    col[holders[1234]] = 1                                            # size 1
    col[holders[2000 + rng.choice(2000, k, replace=False)]] = 2      # exactly k
    col[np.concatenate([holders[:40], others[:110]])] = 3             # 150 matches, 40 with the term
    col[others[200:260]] = 4                                          # matches that hold no query term
    tags = {0: col}
    _load(engine, idx, tags)
    q = idx.term_ids([1])
    conds = [[(0, 0)], [(0, 1)], [(0, 2)], [(0, 3)], [(0, 4)]]
    got = _check(engine, idx, [q] * len(conds), conds, k, tags)
    assert got[2].tolist()[:3] == [0, 1, k]
    if variant == "okapi":
        assert got[2][3] == 40 and got[2][4] == 0
    else:
        assert got[2][3] == k and got[2][4] == 60
        f = be.fast(idx)
        assert (got[1][4][:60] == f.get_scores(list(q))[others[200]]).all()


@pytest.mark.parametrize("variant", VARIANTS)
def test_low_scoring_matches_behind_high_scoring_non_matches(engine, variant):
    """2000 docs hold the query term 5 times (high scores, code 0), 300 docs once (low scores, code 1), spread over every
    range; k = 100 of the low ones.  Fails if the sample pass or the collect pass ignores the filter (module docstring)."""
    n = 4 * be.RANGE + 500
    hi = np.linspace(0, n - 1, 2000).astype(np.int64)
    lo = np.setdiff1d(np.linspace(3, n - 4, 300).astype(np.int64), hi)
    doc = np.concatenate([hi, lo])
    tf = np.concatenate([np.full(len(hi), 5), np.ones(len(lo), np.int64)])
    idx = be.index_from_triples(n, doc, np.full(len(doc), 1), tf, fill=4, variant=variant)
    col = np.full(n, 2, np.int32)
    col[hi] = 0
    col[lo] = 1
    tags = {0: col}
    _load(engine, idx, tags)
    q = idx.term_ids([1])
    got = _check(engine, idx, [q, q, q], [[(0, 1)], [(0, 0)], []], 100, tags)
    assert set(got[0][0].tolist()) <= set(lo.tolist()) and got[2][0] == 100
    f = be.fast(idx)
    s = f.get_scores(list(q))
    assert s[lo].max() < s[hi].min()    # every match scores below every non-match


@pytest.mark.parametrize("variant", VARIANTS)
def test_ties_straddling_rank_k_among_matches(engine, variant):
    case = be.tie_case(3000, variant)
    idx = case.idx
    n = idx.n_docs
    d = np.unique(np.linspace(0, n - 1, 3000).astype(np.int64))
    col = np.full(n, 0, np.int32)
    col[d[::20]] = 1                                     # 150 exactly tied matches, k = 100 cuts inside the tie
    tags = {0: col}
    _load(engine, idx, tags)
    got = _check(engine, idx, case.queries, [[(0, 1)], [(0, 1)]], 100, tags)
    assert got[2][0] == 100 and len(set(got[1][0].tolist())) == 1


@pytest.mark.parametrize("variant", VARIANTS)
def test_queries_longer_than_one_term_block(engine, variant):
    case = be.long_query_case(variant)
    idx = case.idx
    n = idx.n_docs
    tags = {0: (np.arange(n) % 3).astype(np.int32), 1: (np.arange(n) % 4 == 0).astype(np.int32)}
    _load(engine, idx, tags)
    conds = [[(0, 1)] if i % 2 else [(0, 2), (1, 1)] for i in range(len(case.queries))]
    conds[3] = []
    _check(engine, idx, case.queries, conds, case.k, tags)


@pytest.mark.parametrize("variant", VARIANTS)
def test_many_docs_and_queries_several_sub_batches(engine, variant):
    """300 k docs x 1000 queries (several sub-batches), every third query unfiltered."""
    case = be.strip_case(variant)
    idx = case.idx
    n = idx.n_docs
    tags = {0: (np.arange(n) % 10).astype(np.int32), 1: ((np.arange(n) // 512) % 3).astype(np.int32)}
    _load(engine, idx, tags)
    conds = [[] if b % 3 == 0 else ([(0, b % 10)] if b % 3 == 1 else [(0, b % 10), (1, b % 3)])
             for b in range(len(case.queries))]
    _check(engine, idx, case.queries, conds, case.k, tags, rows=case.rows)


@pytest.mark.parametrize("variant", VARIANTS)
def test_device_form_equals_host_form(engine, variant):
    import torch

    idx, qs = _corpus_a(variant)
    tags = _tags_a(idx.n_docs)
    _load(engine, idx, tags)
    queries = [qs[i % len(qs)] for i in range(len(CONDS_A))]
    flat, off = engine.pack_queries(queries)
    f_off, fld, code = fo.csr(CONDS_A)
    want = engine.bm25_topk(queries, 100, filters=(f_off, fld, code))
    dev = lambda a: torch.from_numpy(a).cuda()
    got = engine.bm25_topk_dev(dev(flat), dev(off), len(queries), int(off[-1]), int(np.diff(off).max()), 100,
                               filters=(dev(f_off), dev(fld), dev(code)))
    torch.cuda.synchronize()
    for g, w in zip(got, want):
        g = g.cpu().numpy()
        assert np.array_equal(be.bits(g) if g.dtype == np.float64 else g, be.bits(w) if w.dtype == np.float64 else w)


def test_errors_and_column_lifetime(engine):
    from sentio_b200._lib import SentioB200ArgError, SentioB200Error

    idx, qs = _corpus_a("okapi")
    engine.load_bm25(idx)
    n = idx.n_docs
    engine.load_bm25_tags(0, np.zeros(n, np.int32))
    with pytest.raises(SentioB200ArgError):
        engine.load_bm25_tags(1, np.zeros(n - 1, np.int32))     # wrong column length
    with pytest.raises(SentioB200ArgError):
        engine.load_bm25_tags(16, np.zeros(n, np.int32))        # field out of range
    with pytest.raises(SentioB200ArgError):
        engine.load_bm25_tags(1, np.full(n, -2, np.int32))      # code below -1
    with pytest.raises(SentioB200Error) as e:
        engine.bm25_topk(qs[:2], 10, filters=fo.csr([[(0, 0)], [(1, 0)]]))    # field 1 not loaded
    assert not isinstance(e.value, SentioB200ArgError)
    with pytest.raises(SentioB200ArgError):
        engine.bm25_topk(qs[:1], 10, filters=fo.csr([[(16, 0)]]))
    got = engine.bm25_topk(qs[:1], 10, filters=fo.csr([[(0, 0)]]))
    assert got[2][0] == 10
    engine.load_bm25(idx)                                       # a new index drops the columns
    with pytest.raises(SentioB200Error):
        engine.bm25_topk(qs[:1], 10, filters=fo.csr([[(0, 0)]]))
    got = engine.bm25_topk(qs[:1], 10, filters=fo.csr([[]]))   # no condition: unfiltered, no column needed
    assert got[2][0] == 10
