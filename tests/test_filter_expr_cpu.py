"""query_points filters without a GPU: the compiler (PayloadIndex.compile_programs) against the row-by-row evaluator on
thousands of seeded random filter trees, legacy conjunctions, every refusal and limit, and the store's query_points /
query_batch_points on an oracle engine double."""
import math
from types import SimpleNamespace as NS

import numpy as np
import pytest

from filter_expr_oracle import matches, run_programs
from sentio_b200 import payload_filter as pf

BIG = 2 ** 53
VALUES = [_ for _ in (True, False, 0, 1, -1, 2, BIG, -BIG, 1.0, 0.5, -0.0, 0.0, math.inf, -math.inf, math.nan, "x", "y",
                      "1", None)]
BOUNDS = [-math.inf, -BIG, -1, -0.0, 0, 0.0, 0.5, 1, 1.0, 2, BIG, math.inf]
KEYS = ["a", "b", "m.c"]


def _payloads(rng, n):
    out = []
    for _ in range(n):
        p = {}
        for key in KEYS:
            if rng.random() < 0.8:
                v = VALUES[rng.integers(len(VALUES))]
                if "." in key:
                    p.setdefault("m", {})["c"] = v
                else:
                    p[key] = v
        out.append(p)
    return out


def _leaf(rng):
    key = KEYS[rng.integers(len(KEYS))]
    kind = rng.integers(3)
    if kind == 0:
        v = [True, False, 0, 1, -1, BIG, "x", "y", "1"][rng.integers(9)]
        return NS(key=key, match=NS(value=v), range=None)
    if kind == 1:
        pool = [0, 1, -1, 2, BIG, 7] if rng.random() < 0.5 else ["x", "y", "1", "z"]
        vals = [pool[i] for i in rng.choice(len(pool), size=rng.integers(0, 4), replace=False)]
        return NS(key=key, match=NS(any=vals), range=None)
    r = NS(gt=None, gte=None, lt=None, lte=None)
    for b in ("gt", "gte", "lt", "lte"):
        if rng.random() < 0.4:
            setattr(r, b, BOUNDS[rng.integers(len(BOUNDS))])
    return NS(key=key, match=None, range=r)


def _tree(rng, depth):
    def conds():
        return [_tree(rng, depth + 1) if depth < 3 and rng.random() < 0.25 else _leaf(rng)
                for _ in range(rng.integers(0, 4))]

    f = NS(must=conds() if rng.random() < 0.7 else None, should=conds() if rng.random() < 0.5 else None,
           must_not=conds() if rng.random() < 0.5 else None, min_should=None)
    if rng.random() < 0.2:
        cs = conds()
        f.min_should = NS(conditions=cs, min_count=int(rng.integers(0, len(cs) + 2)))
    return f


class _Cols:
    """The device columns a PayloadIndex would load, kept in NumPy."""

    def __init__(self, payloads):
        self.tags, self.vals = {}, {}
        self.index = pf.PayloadIndex(payloads, self.tags.__setitem__, None, self.vals.__setitem__, None)


def test_random_trees_interpreter_equals_evaluator():
    rng = np.random.default_rng(7)
    checked = 0
    for rnd in range(20):
        payloads = _payloads(rng, 120)
        cols = _Cols(payloads)
        filters = [_tree(rng, 1) for _ in range(100)]
        off, prog, pool = cols.index.compile_programs(filters)
        got = run_programs(off, prog, pool, cols.tags, cols.vals, len(payloads))
        for b, flt in enumerate(filters):
            want = np.array([matches(flt, p) for p in payloads])
            assert np.array_equal(got[b], want), (rnd, b)
            checked += 1
    assert checked == 2000


def test_edge_values_in_ranges():
    payloads = [{"v": v} for v in (-0.0, 0.0, 0, math.inf, -math.inf, math.nan, BIG, -BIG, True, 1, 1.0, "1", None)]
    payloads.append({})
    cols = _Cols(payloads)
    for b in [dict(gte=0), dict(gt=0), dict(lte=-0.0), dict(lt=0.0), dict(gte=math.inf), dict(gt=-math.inf),
              dict(lte=-math.inf), dict(gte=BIG), dict(gt=BIG - 1), dict(), dict(gte=1, lte=1), dict(gt=1, gte=0)]:
        r = NS(gt=None, gte=None, lt=None, lte=None)
        for k, v in b.items():
            setattr(r, k, v)
        flt = NS(must=[NS(key="v", range=r, match=None)])
        off, prog, pool = cols.index.compile_programs([flt])
        got = run_programs(off, prog, pool, cols.tags, cols.vals, len(payloads))[0]
        assert got.tolist() == [matches(flt, p) for p in payloads], b


def test_legacy_filters_give_the_rows_of_compile_filter():
    rng = np.random.default_rng(3)
    payloads = _payloads(rng, 200)
    cols = _Cols(payloads)
    for _ in range(200):
        conds = [(KEYS[rng.integers(3)], [True, 0, 1, "x", "y", BIG][rng.integers(6)]) for _ in range(rng.integers(0, 4))]
        flt = NS(must=[NS(key=k, match=NS(value=v)) for k, v in conds])
        off, prog, pool = cols.index.compile_programs([flt])
        got = run_programs(off, prog, pool, cols.tags, cols.vals, len(payloads))[0]
        f_off, fld, code = cols.index.compile([flt])
        want = np.ones(len(payloads), bool)
        for i in range(f_off[1]):
            want &= (cols.tags[int(fld[i])] == code[i]) if code[i] >= 0 else False
        assert np.array_equal(got, want)
        assert pf.compile_filter(flt) == [(k, v) for k, v in conds]


def test_matchany_unknown_values_drop_out_and_empty_matches_nothing():
    cols = _Cols([{"s": "a"}, {"s": "b"}, {"s": 1}, {}])
    off, prog, pool = cols.index.compile_programs([NS(must=[NS(key="s", match=NS(any=["b", "zz"]))]),
                                                   NS(must=[NS(key="s", match=NS(any=[]))])])
    got = run_programs(off, prog, pool, cols.tags, cols.vals, 4)
    assert got.tolist() == [[False, True, False, False], [False] * 4]
    assert pool.tolist() == [1]


def _fc(key, **match):
    return NS(key=key, match=NS(**match), range=None)


@pytest.mark.parametrize("flt, what", [
    (NS(must=[_fc("a", except_=[1])]), "MatchExcept"),
    (NS(must=[_fc("a", text="x")]), "MatchText"),
    (NS(must=[_fc("a", phrase="x y")]), "MatchPhrase"),
    (NS(must=[NS(is_empty=NS(key="a"))]), "IsEmpty"),
    (NS(must=[NS(is_null=NS(key="a"))]), "IsNull"),
    (NS(must=[NS(has_id=[1])]), "HasId"),
    (NS(must=[NS(nested=NS(key="a", filter=None))]), "NestedCondition"),
    (NS(must=[NS(key="a", geo_radius=NS(), match=None)]), "geo_radius"),
    (NS(must=[NS(key="a", values_count=NS(gt=1), match=None)]), "values_count"),
    (NS(must=[NS(key="a", datetime_range=NS(gt="2020"), match=None)]), "datetime_range"),
    (NS(must=[_fc("a", any=[1, "x"])]), "mixes"),
    (NS(must=[_fc("a", any=[True])]), "bool"),
    (NS(must=[_fc("a", any=list(range(1025)))]), "at most 1024"),
    (NS(must=[NS(key="a", range=NS(gt=True, gte=None, lt=None, lte=None), match=None)]), "non-numeric"),
    (NS(must=[NS(key="a", range=NS(gt="1", gte=None, lt=None, lte=None), match=None)]), "non-numeric"),
    (NS(must=[NS(key="a", range=NS(gt=BIG + 1, gte=None, lt=None, lte=None), match=None)]), "2\\*\\*53"),
    (NS(must=[_fc("a", value=1.5)]), "non-scalar"),
    (NS(must=[_fc("a", value=1)] * 65), "64 conditions"),
    ({"a": 1}, "unsupported filter"),
])
def test_refusals_and_limits_raise(flt, what):
    cols = _Cols([{"a": 1}])
    with pytest.raises(ValueError, match=what):
        cols.index.compile_programs([flt])


def test_depth_and_key_limits():
    f = NS(must=[_fc("a", value=1)])
    for _ in range(7):
        f = NS(must=[f])
    cols = _Cols([{"a": 1}])
    cols.index.compile_programs([f])       # depth 8
    with pytest.raises(ValueError, match="deeper than 8"):
        cols.index.compile_programs([NS(must=[f])])
    cols = _Cols([{f"k{i}": i for i in range(20)}])
    rng = NS(gt=0, gte=None, lt=None, lte=None)
    for i in range(pf.MAX_VALUE_FIELDS):
        cols.index.compile_programs([NS(must=[NS(key=f"k{i}", range=rng, match=None)])])
    with pytest.raises(ValueError, match="range-filtered"):
        cols.index.compile_programs([NS(must=[NS(key="k19", range=rng, match=None)])])
    with pytest.raises(ValueError, match="2\\*\\*53"):
        _Cols([{"n": BIG + 1}]).index.compile_programs([NS(must=[NS(key="n", range=rng, match=None)])])
    with pytest.raises(ValueError, match="list-valued"):
        _Cols([{"n": [1]}]).index.compile_programs([NS(must=[NS(key="n", range=rng, match=None)])])


# ------------------------------------------------------------------------------------------------ the store
class WhereOracleEngine:
    """The B200Engine methods query_points uses, answered in fp64 NumPy over the input vectors."""
    METRICS = {"cosine": 0, "dot": 1, "euclid": 2}
    DATATYPES = {"float16": 0, "float32": 1}

    def __init__(self, device=0):
        self.tags, self.vals = {}, {}

    def close(self):
        pass

    def load_dense(self, vecs, id_base=0, slot=0, metric="cosine", storage="float16"):
        self.x = np.asarray(vecs, np.float64)
        self.metric = metric
        self.tags, self.vals = {}, {}

    def load_dense_tags(self, f, codes, slot=0):
        self.tags[f] = np.asarray(codes, np.int32).copy()

    def load_dense_values(self, f, vals, slot=0):
        self.vals[f] = np.asarray(vals, np.float64).copy()

    def dense_tags_write(self, f, rows, codes, slot=0):
        self.tags[f][np.asarray(rows)] = codes

    def dense_values_write(self, f, rows, vals, slot=0):
        self.vals[f][np.asarray(rows)] = vals

    def dense_upsert(self, rows, vecs, slot=0):
        rows = np.asarray(rows)
        grow = int(rows.max()) + 1 - len(self.x)
        if grow > 0:
            self.x = np.concatenate([self.x, np.zeros((grow, self.x.shape[1]))])
            for d, fill in ((self.tags, -1), (self.vals, np.nan)):
                for f in d:
                    d[f] = np.concatenate([d[f], np.full(grow, fill, d[f].dtype)])
        self.x[rows] = vecs
        for f in self.tags:
            self.tags[f][rows] = -1
        for f in self.vals:
            self.vals[f][rows] = np.nan

    def dense_fetch(self, rows, slot=0):
        return self.x[np.asarray(rows, np.int64)].astype(np.float32)

    def _scores(self, q):
        if self.metric == "euclid":
            return np.sqrt(((self.x - q) ** 2).sum(1))
        s = self.x @ q
        if self.metric == "cosine":
            den = np.linalg.norm(self.x, axis=1) * np.linalg.norm(q)
            s = np.divide(s, den, out=np.zeros_like(s), where=den > 0)
        return s

    def _topk(self, q, k, masks):
        B = len(q)
        ids, sc, cnt = np.full((B, k), -1, np.int64), np.zeros((B, k)), np.zeros(B, np.int32)
        for b in range(B):
            s = self._scores(np.asarray(q[b], np.float64))
            rows = np.flatnonzero(masks[b])
            key = s[rows] if self.metric == "euclid" else -s[rows]
            o = rows[np.lexsort((rows, key))][:k]
            ids[b, :len(o)], sc[b, :len(o)], cnt[b] = o, s[o], len(o)
        return ids, sc, cnt

    def dense_topk(self, q, k, slot=0):
        return self._topk(q, k, np.ones((len(q), len(self.x)), bool))

    def dense_topk_where(self, q, k, programs, slot=0):
        off, prog, pool = programs
        return self._topk(q, k, run_programs(off, prog, pool, self.tags, self.vals, len(self.x)))


@pytest.fixture
def store(monkeypatch):
    from sentio_b200 import vector_store

    monkeypatch.setattr(vector_store, "B200Engine", WhereOracleEngine)
    s = vector_store.B200VectorStore(0)
    rng = np.random.default_rng(11)
    vecs = rng.standard_normal((80, 8)).astype(np.float32)
    payloads = [{"year": 2000 + i % 30, "src": f"s{i % 5}", "public": i % 3 == 0} for i in range(80)]
    for dist in ("Cosine", "Euclid"):
        s.create_collection(dist, vecs, ids=[f"p{i}" for i in range(80)], payloads=payloads,
                            vectors_config=vector_store.VectorParams(8, dist))
    return s, vecs, payloads


def _range(key, **b):
    r = NS(gt=None, gte=None, lt=None, lte=None)
    for k, v in b.items():
        setattr(r, k, v)
    return NS(key=key, range=r, match=None)


@pytest.mark.parametrize("coll", ["Cosine", "Euclid"])
def test_query_points_offset_threshold_and_filters(store, coll):
    s, vecs, payloads = store
    flt = NS(must=[_range("year", gte=2010)], should=[_fc("src", any=["s1", "s2"]), _fc("public", value=True)],
             must_not=[_fc("src", value="s4")])
    q = vecs[3] + 0.1
    want = [f"p{i}" for i in range(80) if matches(flt, payloads[i])]
    full = s.query_points(coll, q, query_filter=flt, limit=80).points
    assert sorted(p.id for p in full) == sorted(want)
    sc = [p.score for p in full]
    assert sc == (sorted(sc) if coll == "Euclid" else sorted(sc, reverse=True))
    page = s.query_points(coll, NS(nearest=q), query_filter=flt, limit=4, offset=3).points
    assert [p.id for p in page] == [p.id for p in full[3:7]]
    t = full[5].score
    kept = s.query_points(coll, q, query_filter=flt, limit=20, score_threshold=t).points
    assert [p.id for p in kept] == [p.id for p in full[:20] if (p.score <= t if coll == "Euclid" else p.score >= t)]
    assert len(kept) >= 6
    vec = s.query_points(coll, q, limit=2, with_vectors=True, with_payload=False).points
    assert vec[0].payload is None and vec[0].vector == s.retrieve(coll, [vec[0].id], with_vectors=True)[0].vector


def test_query_batch_points_is_one_batch_of_single_queries(store):
    s, vecs, _ = store
    reqs = [NS(query=vecs[i], filter=f, limit=lim, offset=off, score_threshold=None, with_payload=True)
            for i, (f, lim, off) in enumerate([(None, 5, 0), (NS(must=[_range("year", lt=2005)]), 3, 2),
                                               (NS(must_not=[_fc("public", value=True)]), 7, None)])]
    got = s.query_batch_points("Cosine", reqs)
    for r, resp in zip(reqs, got):
        one = s.query_points("Cosine", r.query, query_filter=r.filter, limit=r.limit, offset=r.offset)
        assert [(p.id, p.score) for p in resp.points] == [(p.id, p.score) for p in one.points]


def test_query_request_defaults_of_none_read_as_false(store):
    """Qdrant's QueryRequest leaves with_payload and with_vector None unless set; None means False."""
    s, vecs, _ = store
    req = NS(query=vecs[0], filter=NS(must=[_range("year", gte=2010)]), limit=5, offset=None, score_threshold=None,
             with_payload=None, with_vector=None, using=None, prefetch=None, lookup_from=None, params=None)
    got = s.query_batch_points("Cosine", [req])[0].points
    want = s.query_points("Cosine", vecs[0], query_filter=req.filter, limit=5).points
    assert [(p.id, p.score) for p in got] == [(p.id, p.score) for p in want]
    assert all(p.payload is None and p.vector is None for p in got)


@pytest.mark.parametrize("kw, what", [
    (dict(query="p1"), "point id"),
    (dict(query=7), "point id"),
    (dict(query=NS(recommend=NS(positive=["p1"]))), "not supported"),
    (dict(query=NS(fusion="rrf")), "not supported"),
    (dict(query=NS(nearest=[0.0] * 8, mmr=NS(diversity=0.5))), "mmr"),
    (dict(prefetch=[NS()]), "prefetch"),
    (dict(lookup_from=NS(collection="x")), "lookup_from"),
    (dict(using="text"), "using"),
    (dict(limit=1000, offset=25), "1024"),
])
def test_query_points_refusals(store, kw, what):
    s, vecs, _ = store
    args = dict(query=vecs[0])
    args.update(kw)
    with pytest.raises(ValueError, match=what):
        s.query_points("Cosine", **args)


def test_upsert_with_an_inexact_int_leaves_the_collection_unchanged(store):
    s, vecs, _ = store
    flt = NS(must=[_range("year", gte=2020)])
    before = s.query_points("Cosine", vecs[0], query_filter=flt, limit=50).points
    col = s._collections["Cosine"]
    snap = (list(col.ids), [dict(p) for p in col.payloads], {f: v.copy() for f, v in col.engine.vals.items()})
    with pytest.raises(ValueError, match="2\\*\\*53"):
        s.upsert("Cosine", [NS(id="new", vector=vecs[1], payload={"year": BIG + 1})])
    assert col.ids == snap[0] and col.payloads == snap[1]
    assert all(np.array_equal(col.engine.vals[f], v, equal_nan=True) for f, v in snap[2].items())
    after = s.query_points("Cosine", vecs[0], query_filter=flt, limit=50).points
    assert [(p.id, p.score) for p in after] == [(p.id, p.score) for p in before]
    s.upsert("Cosine", [NS(id="p0", vector=vecs[0], payload={"year": 2021.5})])   # values follow upserts
    assert "p0" in {p.id for p in s.query_points("Cosine", vecs[0], query_filter=flt, limit=80).points}


def test_one_filter_object_for_many_queries_compiles_once_and_means_the_same():
    rng = np.random.default_rng(21)
    payloads = _payloads(rng, 150)
    cols = _Cols(payloads)
    f = _tree(rng, 1)
    while parse_free(f):
        f = _tree(rng, 1)
    off, prog, pool = cols.index.compile_programs([f, None, f, f])
    n = off[1] - off[0]
    assert off.tolist() == [0, n, n, 2 * n, 3 * n]
    assert len(pool) == len(cols.index.compile_programs([f])[2])      # the pool codes are shared, not repeated
    got = run_programs(off, prog, pool, cols.tags, cols.vals, len(payloads))
    want = np.array([matches(f, p) for p in payloads])
    assert all(np.array_equal(got[b], want) for b in (0, 2, 3)) and got[1].all()


def parse_free(f):
    """True when the filter compiles to the empty program (no constraint)."""
    return pf.parse_expr(f) is None
