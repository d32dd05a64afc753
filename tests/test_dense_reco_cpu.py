"""Recommendation by example (DESIGN.md K1j) in the store, against a NumPy engine double: strategy parsing, mixed id
and vector examples, id exclusion, refusals that leave the collection unchanged, offset / limit / threshold cuts, the
batch equal to each request alone, and the pinned merge formula."""
import math
from types import SimpleNamespace as NS

import numpy as np
import pytest

from filter_expr_oracle import run_programs
from reco_oracle import best, g, merged, reco_brute, reco_topk


class RecoOracleEngine:
    """The B200Engine methods recommend uses, in fp64 NumPy over the input vectors."""
    METRICS = {"cosine": 0, "dot": 1, "euclid": 2}
    DATATYPES = {"float16": 0, "float32": 1}
    RECO_STRATEGIES = {"average_vector": 0, "best_score": 1, "sum_scores": 2}
    calls = []

    def __init__(self, device=0):
        self.tags, self.vals = {}, {}

    def close(self):
        pass

    def load_dense(self, vecs, id_base=0, slot=0, metric="cosine", storage="float16"):
        self.x = np.asarray(vecs, np.float32).astype(np.float64)
        self.metric = metric

    def load_dense_tags(self, f, codes, slot=0):
        self.tags[f] = np.asarray(codes, np.int32).copy()

    def load_dense_values(self, f, vals, slot=0):
        self.vals[f] = np.asarray(vals, np.float64).copy()

    def dense_fetch(self, rows, slot=0):
        return self.x[np.asarray(rows, np.int64)].astype(np.float32)

    def _masks(self, B, programs):
        if programs is None:
            return np.ones((B, len(self.x)), bool)
        off, prog, pool = programs
        return run_programs(off, prog, pool, self.tags, self.vals, len(self.x))

    def _out(self, per, k):
        B = len(per)
        ids, sc, cnt = np.full((B, k), -1, np.int64), np.zeros((B, k)), np.zeros(B, np.int32)
        for b, (o, s) in enumerate(per):
            ids[b, :len(o)], sc[b, :len(o)], cnt[b] = o, s, len(o)
        return ids, sc, cnt

    def _nearest(self, q, k, masks):
        RecoOracleEngine.calls.append(("topk", len(q)))
        per = []
        for b in range(len(q)):
            cand = np.flatnonzero(masks[b])
            if self.metric == "euclid":
                s = np.sqrt(((self.x - q[b].astype(np.float64)) ** 2).sum(1))
                o = cand[np.lexsort((cand, s[cand]))][:k]
                per.append((o, s[o]))
            else:
                per.append(reco_topk(self.x, None, [q[b]], 1, "sum_scores", self.metric, k, cand))
        return self._out(per, k)

    def dense_topk(self, q, k, slot=0):
        return self._nearest(q, k, self._masks(len(q), None))

    def dense_topk_where(self, q, k, programs, slot=0):
        return self._nearest(q, k, self._masks(len(q), programs))

    def dense_recommend(self, ex, r_off, n_pos, strategies, k, programs=None, slot=0):
        RecoOracleEngine.calls.append(("recommend", len(n_pos)))
        assert self.metric != "euclid" and ex.dtype == np.float32
        masks = self._masks(len(n_pos), programs)
        per = [reco_topk(self.x, None, ex[r_off[r]:r_off[r + 1]], n_pos[r], strategies[r], self.metric, k,
                         np.flatnonzero(masks[r])) for r in range(len(n_pos))]
        return self._out(per, k)


N, D = 60, 6


@pytest.fixture
def store(monkeypatch):
    from sentio_b200 import vector_store

    monkeypatch.setattr(vector_store, "B200Engine", RecoOracleEngine)
    s = vector_store.B200VectorStore(0)
    rng = np.random.default_rng(5)
    vecs = rng.standard_normal((N, D)).astype(np.float32)
    payloads = [{"year": 2000 + i % 20, "src": f"s{i % 4}"} for i in range(N)]
    for dist in ("Cosine", "Dot", "Euclid"):
        s.create_collection(dist, vecs, ids=[f"p{i}" for i in range(N)], payloads=payloads,
                            vectors_config=vector_store.VectorParams(D, dist))
    RecoOracleEngine.calls = []
    return s, vecs, payloads


def test_merge_formula_pinned():
    assert g(0.0) == 0.5 and g(1.0) == 0.75 and g(-1.0) == 0.25
    assert best(0.3, 0.3) == -g(0.3)                       # a tie takes the negative branch
    assert best(0.3, -math.inf) == g(0.3) and best(-math.inf, 0.2) == -g(0.2)
    S = np.array([[0.3, 0.3], [0.5, 0.1], [1.0, -1.0]])
    assert merged(S, 1, "best_score").tolist() == [-g(0.3), g(0.5), 0.75]
    assert merged(S, 1, "sum_scores").tolist() == [0.0, 0.4, 2.0]


@pytest.mark.parametrize("metric", ["cosine", "dot"])
@pytest.mark.parametrize("strategy", ["best_score", "sum_scores"])
def test_oracle_equals_row_by_row_brute_force(metric, strategy):
    rng = np.random.default_rng(1)
    x = rng.standard_normal((40, 5))
    x[3] = 0.0
    ex = rng.standard_normal((4, 5)).astype(np.float32)
    ex[2] = 0.0
    for n_pos in (0, 2, 4):
        i1, s1 = reco_topk(x, None, ex, n_pos, strategy, metric, 40)
        i2, s2 = reco_brute(x, None, ex, n_pos, strategy, metric, 40)
        assert np.allclose(s1, s2, rtol=1e-12, atol=1e-12)
        assert sorted(i1[:10]) == sorted(i2[:10]) or np.allclose(s1[:10], s2[:10], atol=1e-12)


def test_strategy_parsing():
    from sentio_b200.vector_store import RecommendStrategy, parse_strategy

    assert parse_strategy(None) is RecommendStrategy.AVERAGE_VECTOR
    assert parse_strategy("Best_Score") is RecommendStrategy.BEST_SCORE
    assert parse_strategy(NS(name="SUM_SCORES")) is RecommendStrategy.SUM_SCORES
    assert parse_strategy(RecommendStrategy.SUM_SCORES) is RecommendStrategy.SUM_SCORES
    with pytest.raises(ValueError, match="not supported"):
        parse_strategy("max_score")


def _want(s, coll, vecs, pos, neg, strategy, k, metric):
    ex = [vecs[int(e[1:])] if isinstance(e, str) else np.asarray(e, np.float32) for e in pos + neg]
    excl = {int(e[1:]) for e in pos + neg if isinstance(e, str)}
    x = vecs.astype(np.float64)
    if strategy == "average_vector":
        P = np.asarray(ex[:len(pos)], np.float64)
        q = P.mean(0) if not neg else 2 * P.sum(0) / len(P) - np.asarray(ex[len(pos):], np.float64).sum(0) / len(neg)
        ids, sc = reco_topk(x, None, [q.astype(np.float32)], 1, "sum_scores", metric, N)
    else:
        ids, sc = reco_topk(x, None, ex, len(pos), strategy, metric, N)
    return [(f"p{i}", v) for i, v in zip(ids, sc) if i not in excl][:k]


@pytest.mark.parametrize("coll", ["Cosine", "Dot"])
@pytest.mark.parametrize("strategy", ["average_vector", "best_score", "sum_scores"])
def test_mixed_examples_exclusion_and_cuts(store, coll, strategy):
    s, vecs, _ = store
    pos, neg = ["p3", vecs[7] + 0.5, "p11"], [vecs[20], "p30"]
    full = s.recommend(coll, positive=pos, negative=neg, strategy=strategy, limit=N)
    want = _want(s, coll, vecs, pos, neg, strategy, N, coll.lower())
    assert [p.id for p in full] == [w[0] for w in want]
    assert np.allclose([p.score for p in full], [w[1] for w in want], rtol=1e-6)
    assert not {"p3", "p11", "p30"} & {p.id for p in full}
    page = s.recommend(coll, positive=pos, negative=neg, strategy=strategy, limit=5, offset=4)
    assert [p.id for p in page] == [p.id for p in full[4:9]]
    t = full[6].score
    kept = s.recommend(coll, positive=pos, negative=neg, strategy=strategy, limit=20, score_threshold=t)
    assert [p.id for p in kept] == [p.id for p in full[:20] if p.score >= t]
    v = s.recommend(coll, positive=pos, negative=neg, strategy=strategy, limit=2, with_vectors=True,
                    with_payload=False)
    assert v[0].payload is None and v[0].vector == s.retrieve(coll, [v[0].id], with_vectors=True)[0].vector


def test_euclid_average_vector_threshold_is_a_distance(store):
    s, vecs, _ = store
    full = s.recommend("Euclid", positive=["p1", "p2"], negative=["p9"], limit=N)
    assert [p.score for p in full] == sorted(p.score for p in full)
    t = full[4].score
    kept = s.recommend("Euclid", positive=["p1", "p2"], negative=["p9"], limit=30, score_threshold=t)
    assert [p.id for p in kept] == [p.id for p in full[:30] if p.score <= t]


def test_filter_uses_the_query_points_language(store):
    s, vecs, payloads = store
    r = NS(key="year", range=NS(gt=None, gte=2010, lt=None, lte=None), match=None)
    flt = NS(must=[r], must_not=[NS(key="src", match=NS(value="s1"))])
    got = s.recommend("Cosine", positive=["p0"], negative=[vecs[5]], strategy="best_score", query_filter=flt,
                      limit=N)
    ok = {f"p{i}" for i in range(N) if payloads[i]["year"] >= 2010 and payloads[i]["src"] != "s1"} - {"p0"}
    assert {p.id for p in got} == ok


def test_batch_equals_each_request_alone_in_one_call_per_family(store):
    s, vecs, _ = store
    reqs = [NS(positive=["p1"], negative=None, strategy=None, filter=None, limit=4, offset=0, with_payload=True),
            NS(positive=["p2", vecs[4]], negative=["p9"], strategy="best_score", filter=None, limit=6, offset=2),
            NS(positive=None, negative=["p5"], strategy="sum_scores",
               filter=NS(must=[NS(key="src", match=NS(any=["s0", "s2"]))]), limit=3, offset=None),
            NS(positive=[vecs[8]], negative=[vecs[9], "p10"], strategy="average_vector", filter=None, limit=5, offset=0)]
    RecoOracleEngine.calls = []
    got = s.recommend_batch("Dot", reqs)
    assert sorted(RecoOracleEngine.calls) == [("recommend", 2), ("topk", 2)]
    for r, g_ in zip(reqs, got):
        one = s.recommend("Dot", positive=r.positive, negative=r.negative, strategy=r.strategy,
                          query_filter=r.filter, limit=r.limit, offset=r.offset or 0)
        assert [(p.id, p.score) for p in g_] == [(p.id, p.score) for p in one]


@pytest.mark.parametrize("coll, kw, what", [
    ("Cosine", dict(positive=["nope"]), "no point"),
    ("Cosine", dict(positive=[[1.0] * (D + 1)]), "dimension"),
    ("Cosine", dict(positive=[[float("nan")] * D]), "NaN"),
    ("Cosine", dict(positive=[{"text": [1.0] * D}]), "named"),
    ("Cosine", dict(positive=[NS(indices=[1], values=[1.0])]), "sparse"),
    ("Cosine", dict(positive=[[[1.0] * D] * 2]), "multi-vector"),
    ("Cosine", dict(positive=["p1"], using="text"), "using"),
    ("Cosine", dict(positive=["p1"], lookup_from=NS(collection="x")), "lookup_from"),
    ("Euclid", dict(positive=["p1"], strategy="best_score"), "Euclid"),
    ("Euclid", dict(positive=["p1"], strategy="sum_scores"), "Euclid"),
    ("Cosine", dict(), "at least one"),
    ("Cosine", dict(negative=["p1"]), "average_vector needs"),
    ("Cosine", dict(positive=[[1.0] * D] * 257, strategy="sum_scores"), "257 examples"),
    ("Cosine", dict(positive=["p1", "p2"], limit=1000, offset=23), "1025"),
    ("Cosine", dict(positive=["p1"], strategy="max"), "not supported"),
])
def test_refusals_leave_the_collection_unchanged(store, coll, kw, what):
    s, vecs, _ = store
    before = [(r.id, r.vector) for r in s.retrieve(coll, [f"p{i}" for i in range(N)], with_vectors=True)]
    RecoOracleEngine.calls = []
    with pytest.raises(ValueError, match=what):
        s.recommend(coll, **kw)
    assert RecoOracleEngine.calls == []
    assert [(r.id, r.vector) for r in s.retrieve(coll, [f"p{i}" for i in range(N)], with_vectors=True)] == before


def test_engine_without_a_strategy_refuses_it(store, monkeypatch):
    s, _, _ = store
    monkeypatch.setattr(RecoOracleEngine, "RECO_STRATEGIES", {"average_vector": 0})
    with pytest.raises(ValueError, match="not supported by"):
        s.recommend("Cosine", positive=["p1"], strategy="best_score")
    assert s.recommend("Cosine", positive=["p1"], limit=2)
