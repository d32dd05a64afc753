"""Dot / Euclid dense search on the device (DESIGN.md K1e) against the fp64 oracle of tests/metric_oracle.py: both scans,
batch and k sweeps, corpora with spread-out norms, zero rows, duplicates, the zero query, extreme query scales (the 1e30
Euclid query must come back exact through the brute-force fallback), filtered search, in-place mutation bit-identical
to a fresh load, the vector store end to end, and Cosine loaded through the metric entry point bit-identical to
``sb_dense_load``."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from metric_oracle import assert_metric_topk, magnitude, metric_topk, stored_metric

pytestmark = pytest.mark.gpu

N = 20000            # > 8192 rows: both scans are eligible
BS = (1, 3, 16, 17, 256, 260)
KS = (1, 10, 100, 1024)
METRICS = ("dot", "euclid")


def corpus(kind, n, d, seed):
    """Gaussian directions with the given norm distribution, plus zero rows, exact duplicates and rows equal to within
    fp16 (same stored direction, norms one ulp apart)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d))
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    if kind == "uniform":
        nrm = rng.uniform(0.5, 2.0, n)
    elif kind == "loguniform":
        nrm = 10.0 ** rng.uniform(-3.0, 3.0, n)
    else:   # a few huge-norm outliers in a uniform corpus
        nrm = rng.uniform(0.5, 2.0, n)
        nrm[rng.choice(n, 5, replace=False)] = 1e4
    x = (x * nrm[:, None]).astype(np.float32)
    x[[11, n // 2, n - 1]] = 0.0
    x[[100, 101, 102]] = x[99]                       # exact duplicates
    x[200] = x[199] * np.float32(1.0 + 2.0 ** -20)   # equal to within fp16: same y, c one ulp-ish apart
    return x


def queries(x, seed, B=260):
    rng = np.random.default_rng(seed + 1)
    d = x.shape[1]
    q = (rng.standard_normal((B, d)) * rng.uniform(0.5, 2.0, (B, 1))).astype(np.float32)
    y, c = stored_metric(x[5:6])
    q[0] = (c[0] * y[0].astype(np.float64)).astype(np.float32)   # a stored v, rounded to fp32
    q[1] = 0.0                                                     # the zero query
    q[2] = x[99]                                                   # the duplicated row
    q[3] = q[4] * np.float32(1e-30)
    return q


def oracle_all(x, q, metric, kmax, rows=None):
    """[(rows, scores, magnitude) per query]"""
    y, c = stored_metric(x)
    out = []
    for b in range(len(q)):
        wi, ws = metric_topk(y, c, q[b], kmax, metric, rows=rows)
        out.append((wi, ws, magnitude(c, q[b], wi, metric)))
    return out


def check(eng, q, want, metric, what, modes=(1, 2), bs=BS, ks=KS, filters=None):
    for mode in modes:
        eng.dense_set_mode(mode)
        try:
            for B in bs:
                for k in ks:
                    ids, sc, cnt = eng.dense_topk(q[:B], k, filters=filters(B) if filters else None)
                    for b in range(B):
                        wi, ws, mag = want[b][0][:k], want[b][1][:k], want[b][2]
                        assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"{what} mode {mode} B {B} k {k} q {b}",
                                           mag=mag)
        finally:
            eng.dense_set_mode(0)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("kind, d", [("uniform", 100), ("uniform", 256), ("uniform", 1024), ("loguniform", 256),
                                     ("outliers", 256)])
def test_topk_matches_oracle(engine, metric, kind, d):
    x = corpus(kind, N, d, seed=d)
    q = queries(x, seed=d)
    engine.load_dense(x, metric=metric)
    assert engine.dense_metric() == metric
    want = oracle_all(x, q, metric, max(KS))
    check(engine, q, want, metric, f"{metric} {kind} d={d}")
    ids, sc, cnt = engine.dense_topk(q[:16], 10)
    if metric == "euclid":
        # the stored v itself is nearest, at a distance at the fp32 rounding level of the query
        assert ids[0, 0] == 5 and sc[0, 0] <= 1e-6 * np.linalg.norm(q[0])
        # the zero query: the smallest-norm rows, at distance ||v||
        y, c = stored_metric(x)
        nv = c * np.sqrt((y.astype(np.float64) ** 2).sum(1))
        assert np.allclose(sc[1, :cnt[1]], np.sort(nv)[:cnt[1]], rtol=1e-9, atol=1e-300)
    else:
        # the zero query scores 0 everywhere: the first k rows
        assert ids[1].tolist() == list(range(10)) and np.all(sc[1] == 0.0)


@pytest.mark.parametrize("mode", (1, 2))
def test_query_scales(engine, mode):
    x = corpus("uniform", N, 256, seed=3)
    rng = np.random.default_rng(4)
    base = rng.standard_normal(256).astype(np.float32)
    q = np.stack([base] * 16 + [base * np.float32(s) for s in (1e-30, 1e30)]).astype(np.float32)   # B = 18
    for metric in METRICS:
        engine.load_dense(x, metric=metric)
        engine.dense_set_mode(mode)
        try:
            fb0 = engine.fallback_count()
            ids, sc, cnt = engine.dense_topk(q, 100)
            fb = engine.fallback_count() - fb0
        finally:
            engine.dense_set_mode(0)
        want = oracle_all(x, q, metric, 100)
        for b in range(len(q)):
            wi, ws, mag = want[b]
            assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"{metric} mode {mode} q {b}", mag=mag)
        if metric == "dot":   # ranking by <q, v> does not depend on the scale of q
            assert np.array_equal(ids[16], ids[0]) and np.array_equal(ids[17], ids[0])
        else:                 # Euclid ranking does; the 1e30 query is answered by the brute-force kernel
            assert not np.array_equal(ids[16], ids[0])
            assert fb >= 1, "the 1e30 Euclid query must be routed to the exact fallback"


@pytest.mark.parametrize("metric", METRICS)
def test_filtered(engine, metric):
    import torch

    d = 256
    x = corpus("loguniform", N, d, seed=11)
    q = queries(x, seed=11, B=260)
    engine.load_dense(x, metric=metric)
    rows = np.arange(N)
    engine.load_dense_tags(0, np.zeros(N, np.int32))                      # 100 % match code 0
    engine.load_dense_tags(1, (rows % 100).astype(np.int32))              # 1 % match code 0
    engine.load_dense_tags(2, (rows >= 1000).astype(np.int32))            # 1000 rows match code 0: gather path
    for field, match in ((0, rows), (1, rows[rows % 100 == 0]), (2, rows[:1000])):
        def filters(B, field=field):
            return (np.arange(B + 1, dtype=np.int32), np.full(B, field, np.int32), np.zeros(B, np.int32))
        want = oracle_all(x, q, metric, 100, rows=match)
        check(engine, q, want, metric, f"{metric} filtered field {field}", bs=(3, 17, 260), ks=(10, 100),
              filters=filters)
        B = 260
        off, fld, code = (torch.from_numpy(a).cuda() for a in filters(B))
        ids, sc, cnt = engine.dense_topk_dev(torch.from_numpy(q[:B]).cuda(), 100, filters=(off, fld, code))
        torch.cuda.synchronize()
        ids, sc, cnt = ids.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy()
        for b in range(B):
            wi, ws, mag = want[b]
            assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"{metric} _dev field {field} q {b}", mag=mag)


def _same(a, b, q, what):
    assert a.dense_count[0] == b.dense_count[0]
    n = a.dense_count[0]
    assert np.array_equal(a.dense_fetch(np.arange(n)), b.dense_fetch(np.arange(n))), f"{what}: stored rows"
    for mode in (1, 2):
        for B, k in ((3, 10), (256, 100), (260, 1024)):
            a.dense_set_mode(mode)
            b.dense_set_mode(mode)
            try:
                for u, v in zip(a.dense_topk(q[:B], k), b.dense_topk(q[:B], k)):
                    assert np.array_equal(u, v), f"{what}: mode {mode} B {B} k {k} differs from a fresh load"
            finally:
                a.dense_set_mode(0)
                b.dense_set_mode(0)


@pytest.mark.parametrize("metric", METRICS)
def test_mutation_matches_fresh_load(built_lib, metric):
    from sentio_b200.engine import B200Engine

    mut, fresh = B200Engine(0), B200Engine(0)
    try:
        d = 256
        rng = np.random.default_rng(21)
        mirror = corpus("uniform", 12000, d, seed=21)
        q = queries(mirror, seed=21)
        mut.load_dense(mirror, metric=metric)
        # overwrite, then append past the capacity (growth), including a row whose norm raises the slot's bound
        over = rng.choice(12000, 300, replace=False)
        v = corpus("loguniform", 300, d, seed=22)
        mut.dense_upsert(over, v)
        mirror[over] = v
        app = corpus("uniform", 9000, d, seed=23)
        app[17] *= np.float32(1e3)
        mut.dense_upsert(np.arange(12000, 21000), app)
        mirror = np.concatenate([mirror, app])
        fresh.load_dense(mirror, metric=metric)
        _same(mut, fresh, q, f"{metric} after upserts")
        want = oracle_all(mirror, q, metric, 100)
        check(mut, q, want, metric, f"{metric} after upserts", bs=(17, 260), ks=(100,))
        # delete (swap-compaction); the raised bound stays, and stays valid
        dead = rng.choice(len(mirror), 2500, replace=False)
        mf, mt = mut.dense_delete(dead)
        keep = len(mirror) - len(dead)
        m2 = mirror.copy()
        m2[mt] = m2[mf]
        mirror = m2[:keep]
        fresh.load_dense(mirror, metric=metric)
        _same(mut, fresh, q, f"{metric} after delete")
        want = oracle_all(mirror, q, metric, 100)
        check(mut, q, want, metric, f"{metric} after delete", bs=(17, 260), ks=(100,))
        # input validation leaves the slot unchanged
        bad = np.zeros((1, d), np.float32)
        bad[0, 0] = np.inf
        with pytest.raises(ValueError):
            mut.dense_upsert([0], bad)
        if metric == "euclid":
            with pytest.raises(ValueError):
                mut.dense_upsert([0], np.full((1, d), 3e37, np.float32))
        _same(mut, fresh, q, f"{metric} after rejected upserts")
    finally:
        mut.close()
        fresh.close()


def test_cosine_through_the_metric_entry_point_is_unchanged(built_lib):
    from sentio_b200._lib import check as rc_check
    from sentio_b200.engine import B200Engine, _ptr

    a, b = B200Engine(0), B200Engine(0)
    try:
        x = corpus("uniform", N, 256, seed=31)
        q = queries(x, seed=31)
        a.load_dense(x)
        rc_check(b._lib.sb_dense_load_metric(b._h, 0, _ptr(x), N, 256, 0, 0, 0), "sb_dense_load_metric")
        b.dense_dim[0], b.dense_count[0] = 256, N
        assert b.dense_metric() == "cosine"
        _same(a, b, q, "cosine via sb_dense_load_metric")
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("dist", ["Dot", "Euclid"])
def test_vector_store(built_lib, dist):
    from sentio_b200.vector_store import B200VectorStore, Distance, VectorParams

    d = 64
    metric = dist.lower()
    x = corpus("uniform", 3000, d, seed=41)
    s = B200VectorStore(0)
    try:
        s.create_collection("c", vectors_config=VectorParams(d, Distance[dist.upper()]))
        s.upsert("c", [NS(id=f"p{i}", vector=x[i].tolist(), payload={"t": "a" if i % 10 == 0 else "b"})
                       for i in range(3000)])
        info = s.get_collection("c")
        assert info.config.params.vectors.distance.name == dist.upper() and info.points_count == 3000
        s.delete("c", [f"p{i}" for i in range(0, 3000, 7)])
        s.upsert("c", [NS(id="p1", vector=(x[1] * 3).tolist(), payload={"t": "a"})])
        live = {f"p{i}": x[i] for i in range(3000) if i % 7}
        live["p1"] = x[1] * 3
        pa = {pid: ("a" if int(pid[1:]) % 10 == 0 or pid == "p1" else "b") for pid in live}
        ids = list(live)
        X = np.stack([live[i] for i in ids]).astype(np.float32)
        y, c = stored_metric(X)
        rng = np.random.default_rng(42)
        Q = rng.standard_normal((20, d)).astype(np.float32)
        flt = NS(must=[NS(key="t", match=NS(value="a"))])
        rows_a = [j for j, i in enumerate(ids) if pa[i] == "a"]
        batch = s.search_batch("c", Q, limit=10)
        fbatch = s.search_batch("c", Q, limit=10, query_filter=flt)
        pos = {pid: j for j, pid in enumerate(ids)}

        def same(hits, wi, ws, what):   # exact duplicates may sit in another row order than `ids`
            got = np.asarray([pos[h.id] for h in hits], np.int64)
            assert_metric_topk(got, np.asarray([h.score for h in hits]), len(hits), wi, ws, what,
                               mag=magnitude(c, Q[b], wi, metric))

        for b in range(len(Q)):
            wi, ws = metric_topk(y, c, Q[b], 10, metric)
            same(s.search("c", Q[b], limit=10), wi, ws, f"search {b}")
            same(batch[b], wi, ws, f"search_batch {b}")
            wi, ws = metric_topk(y, c, Q[b], 10, metric, rows=rows_a)
            same(s.search("c", Q[b], limit=10, query_filter=flt), wi, ws, f"filtered search {b}")
            same(fbatch[b], wi, ws, f"filtered search_batch {b}")
        rec = s.retrieve("c", ["p1", "p2", "missing"], with_vectors=True)
        assert [r.id for r in rec] == ["p1", "p2"]
        for r in rec:
            j = ids.index(r.id)
            assert np.allclose(r.vector, c[j] * y[j].astype(np.float64), rtol=1e-6, atol=1e-7)
            assert np.allclose(r.vector, live[r.id], rtol=2e-3, atol=2e-3 * np.linalg.norm(live[r.id]))
        with pytest.raises(ValueError, match="Manhattan"):
            s.create_collection("m", vectors_config=VectorParams(d, "Manhattan"))
    finally:
        s.close()


def test_scorers_on_a_dot_collection_match_cosine(built_lib):
    from sentio_b200.document import Document
    from sentio_b200.retrievers.scorers import MMRScorer, SemanticSimilarityScorer
    from sentio_b200.vector_store import B200VectorStore, VectorParams

    d = 64
    x = corpus("uniform", 500, d, seed=51)
    qv = np.random.default_rng(52).standard_normal(d).astype(np.float32)
    emb = NS(embed_sync=lambda t: qv, embed_many_sync=lambda texts: (_ for _ in ()).throw(AssertionError()))
    docs = [Document(text="x", id=str(i)) for i in range(0, 500, 9)]
    s = B200VectorStore(0)
    try:
        s.create_collection("cos", x)
        s.create_collection("dot", x, vectors_config=VectorParams(d, "Dot"))
        for cls in (SemanticSimilarityScorer, MMRScorer):
            a = cls(emb, vector_source=(s, "cos")).score("q", docs)
            b = cls(emb, vector_source=(s, "dot")).score("q", docs)
            assert np.array_equal(np.asarray(a), np.asarray(b)), cls.__name__
    finally:
        s.close()
