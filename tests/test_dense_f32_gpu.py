"""Float32 storage (DESIGN.md K1g) on the device against the fp64 oracle on the vectors as given (tests/f32_oracle.py):
Cosine, Dot and Euclid through both scans with batch and k sweeps, filtered and grouped search, extreme query scales and
the zero query, near-duplicates below fp16 precision (which a float16 slot cannot tell apart), in-place mutation
bit-identical to a fresh load, and the vector store and scorers end to end."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from f32_oracle import f32_magnitude, f32_max_norm, f32_scores, f32_topk, f32_topk_many
from groups_oracle import group_search
from metric_oracle import assert_metric_topk

pytestmark = pytest.mark.gpu

N = 20000            # > 8192 rows: both scans are eligible
METRICS = ("cosine", "dot", "euclid")


def corpus(n, d, seed):
    """Gaussian directions, norms uniform in [0.5, 2], plus zero rows and exact duplicates."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d))
    x *= rng.uniform(0.5, 2.0, (n, 1)) / np.linalg.norm(x, axis=1, keepdims=True)
    x = x.astype(np.float32)
    x[[11, n // 2]] = 0.0
    x[[100, 101]] = x[99]
    return x


def queries(x, seed, B=300):
    rng = np.random.default_rng(seed + 1)
    q = (rng.standard_normal((B, x.shape[1])) * rng.uniform(0.5, 2.0, (B, 1))).astype(np.float32)
    q[0] = x[5]        # a stored vector itself
    q[1] = 0.0         # the zero query
    q[2] = x[99]       # the duplicated row
    return q


def check(eng, x, q, metric, what, modes=(1, 2), bs=(1, 300), ks=(1, 100, 1024), filters=None, rows=None):
    want = f32_topk_many(x, q[:max(bs)], max(ks), metric, rows=rows)
    xmax = f32_max_norm(x)
    for mode in modes:
        eng.dense_set_mode(mode)
        try:
            for B in bs:
                for k in ks:
                    ids, sc, cnt = eng.dense_topk(q[:B], k, filters=filters(B) if filters else None)
                    for b in range(B):
                        wi, ws = want[b][0][:k], want[b][1][:k]
                        assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"{what} mode {mode} B {B} k {k} q {b}",
                                           mag=f32_magnitude(xmax, q[b], metric))
        finally:
            eng.dense_set_mode(0)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", (256, 1024))
def test_topk_matches_oracle(engine, metric, d):
    x = corpus(N, d, seed=d)
    q = queries(x, seed=d)
    engine.load_dense(x, metric=metric, storage="float32")
    assert engine.dense_storage() == "float32" and engine.dense_metric() == metric
    check(engine, x, q, metric, f"{metric} d={d}")
    ids, sc, cnt = engine.dense_topk(q[:2], 10)
    if metric == "euclid":
        assert ids[0, 0] == 5 and sc[0, 0] == 0.0, "a stored vector's own query is at distance exactly 0"
    else:
        assert ids[1].tolist() == list(range(10)) and np.all(sc[1] == 0.0), "the zero query: first k rows, score 0"


@pytest.mark.parametrize("mode", (1, 2))
def test_query_scales(engine, mode):
    d = 256
    x = corpus(N, d, seed=3)
    base = np.random.default_rng(4).standard_normal(d).astype(np.float32)
    scales = (1e-30, 1e-10, 1.0, 1e10, 1e30)
    q = np.stack([base] * 16 + [base * np.float32(s) for s in scales] + [np.zeros(d, np.float32)]).astype(np.float32)
    xmax = f32_max_norm(x)
    for metric in METRICS:
        engine.load_dense(x, metric=metric, storage="float32")
        engine.dense_set_mode(mode)
        try:
            ids, sc, cnt = engine.dense_topk(q, 100)
        finally:
            engine.dense_set_mode(0)
        for b in range(len(q)):
            wi, ws = f32_topk(x, q[b], 100, metric)
            assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"{metric} mode {mode} q {b}",
                               mag=f32_magnitude(xmax, q[b], metric))


@pytest.mark.parametrize("metric", METRICS)
def test_filtered_and_grouped(engine, metric):
    d = 256
    x = corpus(N, d, seed=11)
    q = queries(x, seed=11)
    engine.load_dense(x, metric=metric, storage="float32")
    rows = np.arange(N)
    engine.load_dense_tags(1, (rows % 100).astype(np.int32))              # 1 % match code 0: masked scans
    engine.load_dense_tags(2, (rows >= 1000).astype(np.int32))            # 1000 rows match code 0: gather path
    for field, match in ((1, rows[rows % 100 == 0]), (2, rows[:1000])):
        def filters(B, field=field):
            return (np.arange(B + 1, dtype=np.int32), np.full(B, field, np.int32), np.zeros(B, np.int32))
        check(engine, x, q, metric, f"{metric} filtered field {field}", bs=(3, 300), ks=(10, 100), filters=filters,
              rows=match)
    # grouped: 20-row groups, (limit, group_size) = (10, 3), filtered by field 1 too
    groups = (rows // 20).astype(np.int32)
    engine.load_dense_tags(3, groups)
    qg = q[:20]
    for flt, cand in ((None, None), ((np.arange(21, dtype=np.int32), np.full(20, 1, np.int32),
                                      np.zeros(20, np.int32)), rows[rows % 100 == 0])):
        ng, codes, hits, ids, sc = engine.dense_groups(qg, 3, 10, 3, filters=flt)
        for b in range(len(qg)):
            want = group_search(f32_scores(x, qg[b], metric), groups.tolist(), 10, 3, rows=cand,
                                ascending=metric == "euclid")
            assert int(ng[b]) == len(want), f"{metric} groups q {b}"
            mag = f32_magnitude(f32_max_norm(x), qg[b], metric)
            for g, (code, wh) in enumerate(want):
                assert int(codes[b, g]) == code and int(hits[b, g]) == len(wh), f"{metric} group {g} q {b}"
                assert_metric_topk(ids[b, g], sc[b, g], hits[b, g], [r for r, _ in wh], [s for _, s in wh],
                                   f"{metric} group {g} q {b}", mag=mag)


def _near_duplicates(n_dup, d, seed):
    """n_dup rows that all store the same fp16 row y0 (Cosine: fp16(x / ||x||) == y0) but differ in fp32: y0 plus
    perturbations of at most a tenth of the fp16 spacing of each component."""
    rng = np.random.default_rng(seed)
    u = rng.standard_normal(d)
    y0 = (u / np.linalg.norm(u)).astype(np.float16)
    spacing = np.spacing(np.abs(y0)).astype(np.float64)
    dup = y0.astype(np.float64)[None, :] + rng.uniform(-0.1, 0.1, (n_dup, d)) * spacing[None, :]
    dup = dup.astype(np.float32)
    y = (dup.astype(np.float64) / np.linalg.norm(dup.astype(np.float64), axis=1, keepdims=True)).astype(np.float16)
    assert (y == y0[None, :]).all(), "the cluster must be one fp16 row"
    return dup, y0


@pytest.mark.parametrize("n_dup, fallback", [(300, False), (3000, True)])
def test_near_duplicates_cosine(built_lib, n_dup, fallback):
    from sentio_b200.engine import B200Engine

    d, start = 1024, 5000
    f32, f16 = B200Engine(0), B200Engine(0)
    try:
        x = corpus(N, d, seed=61)
        dup, y0 = _near_duplicates(n_dup, d, seed=62)
        x[start:start + n_dup] = dup
        rng = np.random.default_rng(63)
        q = (y0.astype(np.float32)[None, :] + 0.01 * rng.standard_normal((17, d))).astype(np.float32)   # B = 17: wgmma
        f32.load_dense(x, storage="float32")
        f16.load_dense(x)
        cluster = np.arange(start, start + n_dup)
        # the float16 slot stores one row for the whole cluster: exact ties, broken by ascending row
        assert (f16.dense_fetch(cluster) == f16.dense_fetch(cluster[:1])).all()
        for mode in (1, 2):
            for e in (f32, f16):
                e.dense_set_mode(mode)
            try:
                fb0 = f32.fallback_count()
                ids32, sc32, cnt32 = f32.dense_topk(q, 100)
                fb = f32.fallback_count() - fb0
                ids16, _, _ = f16.dense_topk(q, 100)
            finally:
                for e in (f32, f16):
                    e.dense_set_mode(0)
            for b in range(len(q)):
                wi, ws = f32_topk(x, q[b], 100, "cosine")
                assert set(wi.tolist()) <= set(cluster.tolist())
                assert ids32[b].tolist() == wi.tolist(), f"float32 slot: oracle order, mode {mode} q {b}"
                assert_metric_topk(ids32[b], sc32[b], cnt32[b], wi, ws, f"float32 near-dup mode {mode} q {b}", mag=1.0)
                assert ids16[b].tolist() == cluster[:100].tolist(), f"float16 slot: row order, mode {mode} q {b}"
                assert ids32[b].tolist() != ids16[b].tolist()
            if fallback:
                assert fb >= len(q), f"a window of {n_dup} rows must take the brute-force fallback (mode {mode})"
    finally:
        f32.close()
        f16.close()


def test_euclid_own_vector_first(engine):
    d = 1024
    x = corpus(N, d, seed=71)
    rng = np.random.default_rng(72)
    p = 777
    nb = rng.standard_normal((8, d))
    nb *= 1e-6 / np.linalg.norm(nb, axis=1, keepdims=True)
    x[p + 1:p + 9] = (x[p].astype(np.float64)[None, :] + nb).astype(np.float32)
    engine.load_dense(x, metric="euclid", storage="float32")
    q = np.stack([x[p]] * 17)   # B = 1 and B = 17 (wgmma)
    for mode in (1, 2):
        engine.dense_set_mode(mode)
        try:
            for B in (1, 17):
                ids, sc, cnt = engine.dense_topk(q[:B], 10)
                wi, ws = f32_topk(x, q[0], 10, "euclid")
                for b in range(B):
                    assert ids[b, 0] == p and sc[b, 0] == 0.0
                    assert sorted(ids[b, 1:9].tolist()) == list(range(p + 1, p + 9))
                    assert np.all((sc[b, 1:9] > 5e-7) & (sc[b, 1:9] < 2e-6))
                    assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"mode {mode} B {B}",
                                       mag=f32_magnitude(f32_max_norm(x), q[0], "euclid"))
        finally:
            engine.dense_set_mode(0)


def _same(a, b, q, what):
    assert a.dense_count[0] == b.dense_count[0]
    n = a.dense_count[0]
    assert np.array_equal(a.dense_fetch(np.arange(n)), b.dense_fetch(np.arange(n))), f"{what}: fetch"
    for mode in (1, 2):
        for B, k in ((3, 10), (300, 100)):
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
        rng = np.random.default_rng(81)
        mirror = corpus(12000, d, seed=81)
        q = queries(mirror, seed=81)
        mut.load_dense(mirror, metric=metric, storage="float32")
        # random overwrites, growth past the capacity, deletes, and fp16 input widened exactly
        for step in range(4):
            over = rng.choice(len(mirror), 200, replace=False)
            v = corpus(200, d, seed=100 + step) * np.float32(rng.uniform(0.5, 4.0))
            mut.dense_upsert(over, v)
            mirror[over] = v
            app = corpus(3000, d, seed=200 + step)
            if step == 1:
                app = app.astype(np.float16)
            mut.dense_upsert(np.arange(len(mirror), len(mirror) + len(app)), app)
            mirror = np.concatenate([mirror, app.astype(np.float32)])
            dead = rng.choice(len(mirror), 1500, replace=False)
            mf, mt = mut.dense_delete(dead)
            keep = len(mirror) - len(dead)
            m2 = mirror.copy()
            m2[mt] = m2[mf]
            mirror = m2[:keep]
        fresh.load_dense(mirror, metric=metric, storage="float32")
        _same(mut, fresh, q, f"{metric} after mutations")
        got = mut.dense_fetch(np.arange(len(mirror)))
        if metric == "cosine":
            x64 = mirror.astype(np.float64)
            nrm = np.linalg.norm(x64, axis=1, keepdims=True)
            want = np.divide(x64, nrm, out=np.zeros_like(x64), where=nrm > 0).astype(np.float32)
            assert np.allclose(got, want, rtol=2 ** -23, atol=0.0)
        else:
            assert np.array_equal(got, mirror), "fetch returns x bit for bit"
        check(mut, mirror, q, metric, f"{metric} after mutations", bs=(17, 300), ks=(100,))
        bad = np.zeros((1, d), np.float32)
        bad[0, 0] = np.inf
        with pytest.raises(ValueError):
            mut.dense_upsert([0], bad)
        _same(mut, fresh, q[:3], f"{metric} after a rejected upsert")
    finally:
        mut.close()
        fresh.close()


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid"])
def test_vector_store(built_lib, dist):
    from sentio_b200.vector_store import B200VectorStore, Datatype, VectorParams

    d = 64
    metric = dist.lower()
    x = corpus(3000, d, seed=91)
    s = B200VectorStore(0)
    try:
        s.create_collection("c", vectors_config=VectorParams(d, dist, datatype=Datatype.FLOAT32))
        s.upsert("c", [NS(id=f"p{i}", vector=x[i].tolist(), payload={"t": "a" if i % 10 == 0 else "b", "doc": i // 5})
                       for i in range(3000)])
        info = s.get_collection("c")
        assert info.config.params.vectors.datatype is Datatype.FLOAT32 and info.points_count == 3000
        s.delete("c", [f"p{i}" for i in range(0, 3000, 7)])
        s.upsert("c", [NS(id="p1", vector=(x[1] * 3).tolist(), payload={"t": "a", "doc": 0})])
        live = {f"p{i}": x[i] for i in range(3000) if i % 7}
        live["p1"] = x[1] * 3
        ids = list(live)
        X = np.stack([live[i] for i in ids]).astype(np.float32)
        pos = {pid: j for j, pid in enumerate(ids)}
        doc = {pid: (0 if pid == "p1" else int(pid[1:]) // 5) for pid in ids}
        rng = np.random.default_rng(92)
        Q = rng.standard_normal((10, d)).astype(np.float32)
        flt = NS(must=[NS(key="t", match=NS(value="a"))])
        rows_a = [j for j, i in enumerate(ids) if i == "p1" or (int(i[1:]) % 10 == 0)]
        for b in range(len(Q)):
            mag = f32_magnitude(f32_max_norm(X), Q[b], metric)
            for hits, rows in ((s.search("c", Q[b], limit=10), None),
                               (s.search("c", Q[b], limit=10, query_filter=flt), rows_a)):
                wi, ws = f32_topk(X, Q[b], 10, metric, rows=rows)
                got = np.asarray([pos[h.id] for h in hits], np.int64)
                assert_metric_topk(got, np.asarray([h.score for h in hits]), len(hits), wi, ws, f"search {b}", mag=mag)
            res = s.search_groups("c", Q[b], group_by="doc", limit=5, group_size=2)
            want = group_search(f32_scores(X, Q[b], metric), [doc[i] for i in ids], 5, 2, ascending=metric == "euclid")
            assert [g.id for g in res.groups] == [g for g, _ in want]
            for g, (_, wh) in zip(res.groups, want):
                got = np.asarray([pos[h.id] for h in g.hits], np.int64)
                assert_metric_topk(got, np.asarray([h.score for h in g.hits]), len(g.hits), [r for r, _ in wh],
                                   [sc for _, sc in wh], f"group {g.id} q {b}", mag=mag)
        rec = s.retrieve("c", ["p1", "p2", "missing"], with_vectors=True)
        assert [r.id for r in rec] == ["p1", "p2"]
        for r in rec:
            v = np.asarray(live[r.id], np.float32)
            if metric == "cosine":
                v = (v.astype(np.float64) / np.linalg.norm(v.astype(np.float64))).astype(np.float32)
                assert np.allclose(np.asarray(r.vector, np.float32), v, rtol=2 ** -23, atol=0.0)
            else:
                assert np.array_equal(np.asarray(r.vector, np.float32), v), "retrieve returns x bit for bit"
    finally:
        s.close()


def test_scorers_score_the_stored_float32_vectors(built_lib):
    from sentio_b200.document import Document
    from sentio_b200.retrievers.scorers import MMRScorer, SemanticSimilarityScorer
    from sentio_b200.vector_store import B200VectorStore, VectorParams

    d = 64
    x = corpus(500, d, seed=95)
    qv = np.random.default_rng(96).standard_normal(d).astype(np.float32)
    emb = NS(embed_sync=lambda t: qv, embed_many_sync=lambda texts: (_ for _ in ()).throw(AssertionError()))
    docs = [Document(text="x", id=str(i)) for i in range(1, 500, 9)]
    rows = np.asarray([int(dd.id) for dd in docs])
    s = B200VectorStore(0)
    try:
        s.create_collection("f32", x, vectors_config=VectorParams(d, "Dot", datatype="float32"))
        eng = s.engine_of("f32")
        sem = SemanticSimilarityScorer(emb, weight=1.0, vector_source=(s, "f32")).score("q", docs)
        want = f32_scores(x[rows], qv, "cosine")
        assert np.allclose(sem, want, rtol=1e-12, atol=1e-14)
        # both scorers give what they give on the caller's vectors x re-embedded (the path without a vector source)
        emb_x = NS(embed_sync=lambda t: qv, embed_many_sync=lambda texts: x[rows])
        for cls in (SemanticSimilarityScorer, MMRScorer):
            a = cls(emb, vector_source=(s, "f32")).score("q", docs)
            b = cls(emb_x, engine=eng).score("q", docs)
            assert np.array_equal(np.asarray(a), np.asarray(b)), cls.__name__
    finally:
        s.close()
