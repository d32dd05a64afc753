"""Filtered dense search (sb_dense_topk_filtered): the exact top-k of the rows matching each query's payload conditions,
on both scans, the low-cardinality gather path and the brute-force fallback, plus the B200VectorStore `query_filter`."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from helpers import assert_topk_matches
from oracle import dense as dense_oracle

pytestmark = pytest.mark.gpu

N_OF_D = {256: 40000, 1024: 12000}
BMAX = 260
DUP_IN = (50, 100, 2600)      # rows 100..2599 are exact copies of row 50, all inside field 4 == 0
DUP_OUT = (3000, 3200)        # rows 3001..3199 copy row 3000, all outside field 5 == 0


def _corpus(d):
    n = N_OF_D[d]
    rng = np.random.default_rng(d)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x16 = x.astype(np.float16)
    src, lo, hi = DUP_IN
    x16[lo:hi] = x16[src]
    x16[DUP_OUT[0] + 1:DUP_OUT[1]] = x16[DUP_OUT[0]]
    tags = np.zeros((6, n), np.int32)
    u = rng.random(n)
    tags[1] = np.where(u < 0.30, 0, np.where(u < 0.33, 1, np.where(u < 0.333, 2, 3)))   # 30 %, 3 %, 0.3 %
    perm = rng.permutation(n)
    tags[2] = -1                                                 # absent on most rows
    for code, (a, b) in enumerate([(0, 500), (500, 2549), (2549, 2648), (2648, 2657)]):   # 500, 2049, 99, 9 rows
        tags[2][perm[a:b]] = code
    tags[3] = np.arange(n) % 2
    tags[4] = 1
    tags[4][[src, *range(lo, hi)]] = 0
    tags[5] = 0
    tags[5][DUP_OUT[0] + 1:DUP_OUT[1]] = 1
    q = rng.standard_normal((BMAX, d)).astype(np.float32)
    q[2] = x16[src].astype(np.float32)
    q[3] = x16[DUP_OUT[0]].astype(np.float32)
    q[4] = 0.0
    return x16, tags, q


@pytest.fixture(scope="module", params=[256, 1024])
def corpus(request):
    d = request.param
    x16, tags, q = _corpus(d)
    x = x16.astype(np.float64)
    q64 = q.astype(np.float64)
    den = np.sqrt((x * x).sum(1))[:, None] * np.sqrt((q64 * q64).sum(1))[None, :]
    s = np.zeros((len(x), len(q)))
    np.divide(x @ q64.T, den, out=s, where=den > 0)
    return SimpleCorpus(x16, tags, q, s)


class SimpleCorpus:
    def __init__(self, x16, tags, q, s):
        self.x16, self.tags, self.q, self.s = x16, tags, q, s


def _km1(k):   # a condition that exactly k - 1 rows satisfy (k = 1: none)
    return [(2, {1: 99, 10: 3, 100: 2}[k])]


CASES = {
    "all": lambda k: [(0, 0)],
    "p30": lambda k: [(1, 0)],
    "p3": lambda k: [(1, 1)],
    "p0.3": lambda k: [(1, 2)],
    "c500": lambda k: [(2, 0)],
    "k-1": _km1,
    "c2049": lambda k: [(2, 1)],
    "unknown": lambda k: [(1, -1)],
    "conj": lambda k: [(1, 0), (3, 1)],
    "dup_out": lambda k: [(5, 0)],
}


def _csr(conds):
    off = np.zeros(len(conds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in conds])
    fld = np.asarray([f for c in conds for f, _ in c], np.int32)
    code = np.asarray([v for c in conds for _, v in c], np.int32)
    return off, fld, code


def _mask(tags, conds):
    m = np.ones(tags.shape[1], bool)
    for f, v in conds:
        m &= (tags[f] == v) if v >= 0 else False
    return m


def _want(c, b, conds, k):
    idx = np.flatnonzero(_mask(c.tags, conds))
    s = c.s[idx, b]
    o = np.lexsort((idx, -s))[:k]
    return idx[o], s[o]


def _check(c, conds_per_query, k, ids, sc, cnt, what):
    for b, conds in enumerate(conds_per_query):
        wi, ws = _want(c, b, conds, k)
        assert_topk_matches(ids[b], sc[b], cnt[b], wi, ws, what=f"{what} b={b}")
        assert np.all(ids[b, int(cnt[b]):] == -1)


def _load(engine, c):
    engine.load_dense(c.x16)
    for f in range(c.tags.shape[0]):
        engine.load_dense_tags(f, c.tags[f])


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("B", [1, 5, 16, 40, 260])
def test_filtered_topk_matches_oracle(engine, corpus, mode, B):
    c = corpus
    _load(engine, c)
    engine.dense_set_mode(mode)
    try:
        q = c.q[:B]
        for k in (1, 10, 100):
            for name, case in CASES.items():
                conds = [case(k)] * B
                ids, sc, cnt = engine.dense_topk(q, k, filters=_csr(conds))
                _check(c, conds, k, ids, sc, cnt, f"mode={mode} B={B} k={k} {name}")
            names = list(CASES)
            mixed = [[] if b % 7 == 3 else CASES[names[b % len(names)]](k) for b in range(B)]
            ids, sc, cnt = engine.dense_topk(q, k, filters=_csr(mixed))
            _check(c, mixed, k, ids, sc, cnt, f"mode={mode} B={B} k={k} mixed")
    finally:
        engine.dense_set_mode(0)


@pytest.mark.parametrize("mode", [1, 2])
def test_duplicates_inside_the_match_set_take_the_exact_fallback(engine, corpus, mode):
    """More than 2048 exact copies of the query inside the matching set: the window cannot be served, the query goes to
    brute force (the fallback counter says so) and the answer is still exact."""
    c = corpus
    _load(engine, c)
    B = 1 if mode == 1 else 16
    q = np.repeat(c.q[2:3], B, axis=0)
    conds = [[(4, 0)]] * B
    engine.dense_set_mode(mode)
    try:
        before = engine.fallback_count()
        ids, sc, cnt = engine.dense_topk(q, 10, filters=_csr(conds))
        assert engine.fallback_count() > before
    finally:
        engine.dense_set_mode(0)
    src, lo, hi = DUP_IN
    want = np.asarray([src, *range(lo, lo + 9)])
    for b in range(B):
        assert cnt[b] == 10 and np.array_equal(ids[b], want)


def test_duplicates_outside_the_match_set_never_leak(engine, corpus):
    c = corpus
    _load(engine, c)
    for B, mode in ((1, 1), (16, 2)):
        engine.dense_set_mode(mode)
        try:
            q = np.repeat(c.q[3:4], B, axis=0)
            ids, sc, cnt = engine.dense_topk(q, 100, filters=_csr([[(5, 0)]] * B))
        finally:
            engine.dense_set_mode(0)
        assert ids[0, 0] == DUP_OUT[0]
        assert not np.isin(ids[:, :], np.arange(DUP_OUT[0] + 1, DUP_OUT[1])).any()


def test_zero_query_gives_first_matching_rows(engine, corpus):
    c = corpus
    _load(engine, c)
    for B, mode, conds in ((1, 1, [(1, 0)]), (16, 2, [(1, 0)]), (16, 2, [(2, 0)])):
        q = np.zeros((B, c.q.shape[1]), np.float32)
        engine.dense_set_mode(mode)
        try:
            ids, sc, cnt = engine.dense_topk(q, 50, filters=_csr([conds] * B))
        finally:
            engine.dense_set_mode(0)
        want = np.flatnonzero(_mask(c.tags, conds))[:50]
        for b in range(B):
            assert cnt[b] == 50 and np.array_equal(ids[b], want) and np.all(sc[b] == 0.0)


def test_no_conditions_equals_unfiltered(engine, corpus):
    c = corpus
    _load(engine, c)
    for B in (5, 40):
        q = c.q[:B]
        plain = engine.dense_topk(q, 100)
        filt = engine.dense_topk(q, 100, filters=_csr([[]] * B))
        for a, b in zip(plain, filt):
            assert np.array_equal(a, b)


def test_filtered_dev_matches_host(engine, corpus):
    import torch

    c = corpus
    _load(engine, c)
    names = list(CASES)
    conds = [[] if b % 7 == 3 else CASES[names[b % len(names)]](10) for b in range(40)]
    off, fld, code = _csr(conds)
    host = engine.dense_topk(c.q[:40], 10, filters=(off, fld, code))
    dev = [torch.from_numpy(a).cuda() for a in (off, fld, code)]
    out = engine.dense_topk_dev(torch.from_numpy(c.q[:40]).cuda(), 10, filters=tuple(dev))
    torch.cuda.synchronize()
    for a, b in zip(host, out):
        assert np.array_equal(a, b.cpu().numpy())


# ------------------------------------------------------------------------------------------------ B200VectorStore
def _fc(key, value):
    return NS(key=key, match=NS(value=value))


@pytest.fixture(scope="module")
def store(built_lib):
    from sentio_b200.vector_store import B200VectorStore

    rng = np.random.default_rng(7)
    n, d = 10000, 128
    vecs = rng.standard_normal((n, d)).astype(np.float32)
    payloads = []
    for i in range(n):
        md = {"source": f"doc{i % 40}.pdf", "page": int(i % 13), "flag": bool(i % 3 == 0)}
        if i % 5 == 0:
            md["page"] = True if i % 10 == 0 else 1    # True and 1 are different values
        if i % 17 == 0:
            del md["source"]                            # missing key
        payloads.append({"content": f"text {i}", "metadata": md})
    s = B200VectorStore(0)
    s.create_collection("c", vecs, payloads=payloads)
    yield s, vecs, payloads
    s.close()


def _satisfies(payload, conds):
    for key, value in conds:
        cur = payload
        for part in key.split("."):
            if not isinstance(cur, dict) or part not in cur:
                return False
            cur = cur[part]
        if type(cur) is not type(value) or cur != value:
            return False
    return True


def test_store_filters_are_exact(store):
    s, vecs, payloads = store
    rng = np.random.default_rng(3)
    q = rng.standard_normal((20, vecs.shape[1])).astype(np.float32)
    rows16 = dense_oracle.stored_rows(vecs)
    filters = [
        ([("metadata.source", "doc3.pdf")], _fc("metadata.source", "doc3.pdf")),
        ([("metadata.page", 1)], NS(must=[_fc("metadata.page", 1)])),
        ([("metadata.page", True)], NS(must=[_fc("metadata.page", True)])),
        ([("metadata.flag", True), ("metadata.source", "doc7.pdf")],
         NS(must=[_fc("metadata.flag", True), _fc("metadata.source", "doc7.pdf")], should=None, must_not=None)),
        ([("metadata.source", "nope.pdf")], _fc("metadata.source", "nope.pdf")),
        ([("source", "doc3.pdf")], _fc("source", "doc3.pdf")),   # top-level key: absent everywhere
    ]
    for conds, flt in filters:
        match = np.asarray([_satisfies(p, conds) for p in payloads])
        idx = np.flatnonzero(match)
        for b in range(3):
            hits = s.search("c", q[b], limit=25, query_filter=flt)
            assert all(_satisfies(h.payload, conds) for h in hits)
            wi, ws = dense_oracle.dense_topk(rows16[idx], q[b], 25) if len(idx) else ([], [])
            assert [h.id for h in hits] == [str(int(idx[i])) for i in wi]
        batch = s.search_batch("c", q, limit=25, query_filter=flt)
        assert [[h.id for h in r] for r in batch[:3]] == \
            [[h.id for h in s.search("c", q[b], limit=25, query_filter=flt)] for b in range(3)]
    # True and 1 select disjoint rows
    t = {h.id for h in s.search("c", q[0], limit=500, query_filter=_fc("metadata.page", True))}
    o = {h.id for h in s.search("c", q[0], limit=500, query_filter=_fc("metadata.page", 1))}
    assert t and o and not (t & o)


def test_store_per_query_filters_and_none(store):
    s, vecs, payloads = store
    q = np.random.default_rng(4).standard_normal((4, vecs.shape[1])).astype(np.float32)
    flts = [None, _fc("metadata.source", "doc1.pdf"), NS(must=[]), _fc("metadata.flag", False)]
    got = s.search_batch("c", q, limit=10, query_filter=flts)
    for b, f in enumerate(flts):
        assert [h.id for h in got[b]] == [h.id for h in s.search("c", q[b], limit=10, query_filter=f)]
    plain = s.search_batch("c", q, limit=10)
    assert [[(h.id, h.score) for h in r] for r in plain] == \
        [[(h.id, h.score) for h in r] for r in s.search_batch("c", q, limit=10, query_filter=None)]
    assert [(h.id, h.score) for h in s.search("c", q[0], limit=10)] == \
        [(h.id, h.score) for h in got[0]]


@pytest.mark.parametrize("flt", [
    NS(must=[_fc("metadata.page", 1)], should=[_fc("metadata.page", 2)]),
    NS(must=None, must_not=[_fc("metadata.page", 2)]),
    NS(must=[NS(key="metadata.page", range=NS(gte=1), match=None)]),
    NS(must=[NS(key="metadata.page", match=NS(any=[1, 2]))]),
    NS(must=[NS(must=[_fc("metadata.page", 1)])]),
    NS(must=[_fc("metadata.page", 1.5)]),
    NS(must=[_fc("metadata.page", [1])]),
])
def test_store_unsupported_filters_raise(store, flt):
    s, vecs, _ = store
    with pytest.raises(ValueError):
        s.search("c", vecs[0], limit=5, query_filter=flt)
