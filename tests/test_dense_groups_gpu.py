"""Grouped dense search (sb_dense_groups / B200VectorStore.search_groups) against the walk-the-sorted-list oracle:
Cosine, Dot and Euclid; one query and a batch past the 256-query chunk; group-size mixes; a dominant group that forces an
exclusion round; completions through the gather path and the scan path; filters; mutation; duplicates; the zero query."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from groups_oracle import group_search
from metric_oracle import metric_scores, stored_metric

pytestmark = pytest.mark.gpu

N, D = 24000, 256
F_MIX, F_GIANT, F_SINGLE, F_FILTER, F_DOM, F_DUP = range(6)
DOM_ROWS = 1500            # rows of the dominant group (code 0 of F_DOM), clustered around the first query
DUP_SRC, DUP_ROWS = 50, range(100, 110)   # rows 100..109 copy row 50, each in its own F_DUP group


def _corpus():
    rng = np.random.default_rng(7)
    x = rng.standard_normal((N, D)).astype(np.float32)
    x *= rng.uniform(0.5, 2.0, (N, 1)).astype(np.float32)     # spread norms for Dot / Euclid
    # rows have norms ~16 x [0.5, 2]; the cluster sits at norm 24 with spread 0.4 of that, so it holds the nearest rows
    # of the first query under every metric while its scores stay spread out
    center = rng.standard_normal(D).astype(np.float32)
    center *= 24.0 / np.linalg.norm(center)
    dom = rng.permutation(N)[:DOM_ROWS]
    x[dom] = center + 9.6 * rng.standard_normal((DOM_ROWS, D)).astype(np.float32) / np.sqrt(D)
    x[DUP_SRC] *= 36.0 / np.linalg.norm(x[DUP_SRC])            # the best Dot score of its own query
    x[list(DUP_ROWS)] = x[DUP_SRC]
    tags = np.zeros((6, N), np.int32)
    tags[F_MIX] = rng.integers(0, N // 20, N)
    tags[F_MIX][rng.random(N) < 0.05] = -1                     # rows missing the key
    tags[F_GIANT] = np.arange(N)
    tags[F_GIANT][rng.permutation(N)[:3000]] = 0               # one 3000-row group, the rest singletons
    tags[F_SINGLE] = np.arange(N)
    tags[F_FILTER] = np.arange(N) % 3
    tags[F_DOM] = 1 + rng.integers(0, N // 20, N)
    tags[F_DOM][dom] = 0
    tags[F_DUP] = np.arange(N) // 7 + 1
    tags[F_DUP][DUP_SRC] = 0
    tags[F_DUP][list(DUP_ROWS)] = N + np.arange(10)
    q = rng.standard_normal((310, D)).astype(np.float32)
    q[0] = center + 0.8 * rng.standard_normal(D).astype(np.float32) / np.sqrt(D)
    q[1] = x[DUP_SRC]
    return x, tags, q, dom


@pytest.fixture(scope="module")
def corpus():
    x, tags, q, dom = _corpus()
    return NS(x=x, tags=tags, q=q, dom=dom, y=stored_metric(x))


def _scores(c, metric, qv):
    y, cf = c.y
    if metric == "cosine":
        y64 = y.astype(np.float64)
        q64 = np.asarray(qv, np.float32).astype(np.float64)
        den = np.sqrt((y64 * y64).sum(1)) * np.sqrt(q64 @ q64)
        s = np.zeros(len(y64))
        np.divide(y64 @ q64, den, out=s, where=den > 0)
        return s
    return metric_scores(y, cf, qv, metric)


@pytest.fixture(scope="module", params=["cosine", "dot", "euclid"])
def loaded(request, engine, corpus):
    metric = request.param
    engine.load_dense(corpus.x, metric=metric)
    for f in range(corpus.tags.shape[0]):
        engine.load_dense_tags(f, corpus.tags[f])
    return NS(metric=metric, c=corpus)


def _want(c, metric, qv, field, L, G, rows=None):
    groups = [int(g) if g >= 0 else None for g in c.tags[field]]
    return group_search(_scores(c, metric, qv), groups, L, G, rows=rows, ascending=metric == "euclid")


def _check(got, b, want, what):
    ng, codes, hits, ids, sc = got
    assert int(ng[b]) == len(want), f"{what}: {int(ng[b])} groups, want {len(want)}"
    for g, (code, rows) in enumerate(want):
        assert int(codes[b, g]) == code, f"{what}: group {g} is {int(codes[b, g])}, want {code}"
        assert int(hits[b, g]) == len(rows), f"{what}: group {g} has {int(hits[b, g])} hits, want {len(rows)}"
        assert list(map(int, ids[b, g, :len(rows)])) == [r for r, _ in rows], f"{what}: group {g} rows"
        ws = np.array([s for _, s in rows])
        assert np.allclose(sc[b, g, :len(rows)], ws, rtol=1e-9, atol=1e-12 * max(1.0, float(np.abs(ws).max()))), \
            f"{what}: group {g} scores"
        assert np.all(ids[b, g, len(rows):] == -1)
    assert np.all(codes[b, len(want):] == -1)


@pytest.mark.parametrize("B", [1, 300])
@pytest.mark.parametrize("L,G", [(1, 1), (10, 3), (1024, 1)])
@pytest.mark.parametrize("field", [F_MIX, F_SINGLE])
def test_groups_match_oracle(engine, loaded, B, L, G, field):
    c, metric = loaded.c, loaded.metric
    q = c.q[2:2 + B]
    fb0 = engine.fallback_count()
    got = engine.dense_groups(q, field, L, G)
    assert engine.fallback_count() == fb0
    for b in range(0, B, 1 if B == 1 else 37):
        _check(got, b, _want(c, metric, q[b], field, L, G), f"{metric} field={field} L={L} G={G} b={b}")


@pytest.mark.parametrize("L,G", [(3, 2), (10, 3), (20, 1)])
def test_dominant_group_runs_an_exclusion_round(engine, loaded, L, G):
    c, metric = loaded.c, loaded.metric
    q = c.q[:1]
    engine.profile(True)
    try:
        engine.profile_read("dense_group_collect")
        fb0 = engine.fallback_count()
        got = engine.dense_groups(q, F_DOM, L, G)
        n_collect, _ = engine.profile_read("dense_group_collect")
    finally:
        engine.profile(False)
    assert n_collect >= 2, "round 1 held only the dominant group: an exclusion round must have run"
    assert engine.fallback_count() == fb0
    want = _want(c, metric, q[0], F_DOM, L, G)
    assert want[0][0] == 0
    _check(got, 0, want, f"{metric} dominant L={L} G={G}")


def test_completion_through_gather_and_scan(engine, loaded):
    """G = 200 > the hits a 1024-row prefix holds: the 3000-row group completes through the masked scan, the
    singletons through the gather path."""
    c, metric = loaded.c, loaded.metric
    picked = []   # queries whose first 5 groups include the giant group
    for qv in c.q[5:]:
        want = _want(c, metric, qv, F_GIANT, 5, 200)
        if any(code == 0 for code, _ in want):
            picked.append((qv, want))
        if len(picked) == 4:
            break
    q = np.stack([qv for qv, _ in picked])
    engine.profile(True)
    try:
        engine.profile_read("dense_group_assemble")
        got = engine.dense_groups(q, F_GIANT, 5, 200)
        n_asm, _ = engine.profile_read("dense_group_assemble")
    finally:
        engine.profile(False)
    assert n_asm >= 1
    for b, (_, want) in enumerate(picked):
        _check(got, b, want, f"{metric} giant b={b}")


def test_filtered_groups(engine, loaded):
    c, metric = loaded.c, loaded.metric
    B = 40
    q = c.q[10:10 + B]
    conds = [[(F_FILTER, b % 3)] if b % 4 else [] for b in range(B)]
    off = np.zeros(B + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in conds])
    fld = np.asarray([f for x in conds for f, _ in x], np.int32)
    code = np.asarray([v for x in conds for _, v in x], np.int32)
    got = engine.dense_groups(q, F_MIX, 10, 3, filters=(off, fld, code))
    for b in range(B):
        rows = np.flatnonzero(c.tags[F_FILTER] == b % 3) if conds[b] else None
        _check(got, b, _want(c, metric, q[b], F_MIX, 10, 3, rows=rows), f"{metric} filtered b={b}")
    # a condition nothing matches: no groups
    none = engine.dense_groups(q[:1], F_MIX, 10, 3, filters=(np.array([0, 1], np.int32), np.array([F_FILTER], np.int32),
                                                              np.array([7], np.int32)))
    assert int(none[0][0]) == 0


def test_duplicates_across_groups_and_zero_query(engine, loaded):
    c, metric = loaded.c, loaded.metric
    q = np.stack([c.q[1], np.zeros(D, np.float32)])
    got = engine.dense_groups(q, F_DUP, 12, 2)
    want = _want(c, metric, q[0], F_DUP, 12, 2)
    # the source row and its 10 copies score identically: one group each, in row order
    assert [rows[0][0] for _, rows in want[:11]] == [DUP_SRC, *DUP_ROWS]
    _check(got, 0, want, f"{metric} duplicates")
    _check(got, 1, _want(c, metric, q[1], F_DUP, 12, 2), f"{metric} zero query")


def test_fewer_groups_than_limit(engine):
    rng = np.random.default_rng(3)
    x = rng.standard_normal((500, 64)).astype(np.float32)
    tags = np.full(500, -1, np.int32)
    tags[:40] = np.arange(40) % 4   # 4 groups of 10 rows, the rest in no group
    engine.load_dense(x, slot=1)
    engine.load_dense_tags(0, tags, slot=1)
    q = rng.standard_normal((2, 64)).astype(np.float32)
    ng, codes, hits, ids, sc = engine.dense_groups(q, 0, 10, 20, slot=1)
    c = NS(x=x, tags=tags[None, :], y=stored_metric(x))
    for b in range(2):
        assert int(ng[b]) == 4
        _check((ng, codes, hits, ids, sc), b, _want(c, "cosine", q[b], 0, 10, 20), f"few b={b}")


def test_invalid_arguments_raise(engine):
    import ctypes as C

    from sentio_b200._lib import check

    rng = np.random.default_rng(4)
    x = rng.standard_normal((100, 64)).astype(np.float32)
    engine.load_dense(x, slot=1)
    engine.load_dense_tags(0, np.arange(100, dtype=np.int32) % 5, slot=1)
    q = x[:1]
    for L, G in [(0, 1), (1, 0), (1025, 1), (1, 1025)]:
        with pytest.raises(ValueError):
            engine.dense_groups(q, 0, L, G, slot=1)
        # the C ABI refuses the same bounds itself (SB_ERR_ARG -> ValueError)
        out = [np.zeros(4, np.int64) for _ in range(5)]
        p = [a.ctypes.data_as(C.c_void_p) for a in out]
        with pytest.raises(ValueError):
            check(engine._lib.sb_dense_groups(engine._h, 1, q.ctypes.data_as(C.c_void_p), 1, 0, L, G, None, None, None,
                                              *p), "sb_dense_groups")
    with pytest.raises(ValueError):
        engine.dense_groups(q, 16, 1, 1, slot=1)


def _point(pid, vec, payload):
    return NS(id=pid, vector=list(map(float, vec)), payload=payload)


def _store_want(ids, vecs, payloads, qv, key, L, G, allowed=None):
    """Oracle over the store's current points (ids in row order): groups keyed by the typed payload value."""
    from sentio_b200.payload_filter import _MISSING, payload_value, value_key

    y, _ = stored_metric(np.asarray(vecs, np.float32))
    c = NS(y=(y, None))
    groups = []
    for p in payloads:
        v = payload_value(p, key)
        groups.append(None if v is _MISSING or v is None else value_key(v))
    rows = None if allowed is None else [i for i, p in enumerate(payloads) if allowed(p)]
    want = group_search(_scores(c, "cosine", qv), groups, L, G, rows=rows)
    return [(g[1], [(ids[r], s) for r, s in hits]) for g, hits in want]


def _same(res, want):
    assert [g.id for g in res.groups] == [g for g, _ in want]
    for g, (_, hits) in zip(res.groups, want):
        assert [h.id for h in g.hits] == [i for i, _ in hits]
        assert np.allclose([h.score for h in g.hits], [s for _, s in hits], rtol=1e-9, atol=1e-12)


def test_vector_store_search_groups():
    from sentio_b200.vector_store import B200VectorStore

    rng = np.random.default_rng(11)
    n, d = 3000, 128
    vecs = rng.standard_normal((n, d)).astype(np.float32)
    parents = [True, 1, "doc-a", "doc-b", 2, False]
    payloads = []
    for i in range(n):
        md = {"source": f"s{i % 2}"}
        if i % 17:
            md["parent_id"] = parents[i % len(parents)] if i < 600 else f"doc-{i // 10}"
        payloads.append({"content": f"c{i}", "metadata": md})
    ids = [str(i) for i in range(n)]
    store = B200VectorStore(0)
    try:
        store.create_collection("g", vectors=vecs, ids=ids, payloads=payloads)
        q = rng.standard_normal(d).astype(np.float32)
        res = store.search_groups("g", q, group_by="metadata.parent_id", limit=8, group_size=3)
        _same(res, _store_want(ids, vecs, payloads, q, "metadata.parent_id", 8, 3))
        # True and 1 are different groups
        res = store.search_groups("g", q, group_by="metadata.parent_id", limit=400, group_size=1)
        got = [(type(g.id), g.id) for g in res.groups]
        assert (bool, True) in got and (int, 1) in got
        # with a filter
        flt = NS(must=[NS(key="metadata.source", match=NS(value="s1"))])
        res = store.search_groups("g", q, group_by="metadata.parent_id", limit=8, group_size=3, query_filter=flt)
        _same(res, _store_want(ids, vecs, payloads, q, "metadata.parent_id", 8, 3,
                               allowed=lambda p: p["metadata"]["source"] == "s1"))
        # after upsert and delete have moved rows
        new = rng.standard_normal((50, d)).astype(np.float32)
        pts = [_point(str(n + i), new[i], {"content": "n", "metadata": {"source": "s0", "parent_id": "doc-new"}})
               for i in range(50)]
        pts.append(_point("5", new[0] * 2, {"content": "o", "metadata": {"source": "s1", "parent_id": 1}}))
        store.upsert("g", pts)
        store.delete("g", [str(i) for i in range(0, 600, 7)])
        recs = store.scroll("g", limit=10 ** 6)[0]
        cur_ids = [r.id for r in recs]
        cur_pl = [r.payload for r in recs]
        vec_of = {ids[i]: vecs[i] for i in range(n)}
        vec_of.update({str(n + i): new[i] for i in range(50)})
        vec_of["5"] = new[0] * 2
        cur_vecs = np.stack([vec_of[i] for i in cur_ids])
        for qq in (q, new[3]):
            res = store.search_groups("g", qq, group_by="metadata.parent_id", limit=10, group_size=4)
            _same(res, _store_want(cur_ids, cur_vecs, cur_pl, qq, "metadata.parent_id", 10, 4))
        # refused arguments
        for kw in ({"with_lookup": "other"}, {"score_threshold": 0.5}, {"limit": 0}, {"group_size": 2000}):
            with pytest.raises(ValueError):
                store.search_groups("g", q, group_by="metadata.parent_id", **kw)
        store.upsert("g", [_point("x", new[1], {"metadata": {"tags": ["a", "b"]}})])
        with pytest.raises(ValueError):
            store.search_groups("g", q, group_by="metadata.tags")
    finally:
        store.close()
