"""Uint8 storage (DESIGN.md K1i) on the device against the fp64 oracle on the integer vectors (tests/u8_oracle.py):
Cosine, Dot and Euclid across dimensions, row counts, batch sizes and k, every scan mode giving the same bytes, uniform,
clustered, zero, all-255, duplicated and sparse rows, query scales from 1e-30 to 1e30 and the zero query, filtered and
grouped search, in-place mutation byte-identical to a fresh load, SB_U8 input equal to float input, the scorers with a
vector source, the exact fallback of a large duplicate cluster, the _dev entry point, and the vector store."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from groups_oracle import group_search
from metric_oracle import assert_metric_topk
from u8_oracle import clustered_corpus, u8_magnitude, u8_scores, u8_topk, u8_topk_many

pytestmark = pytest.mark.gpu

METRICS = ("cosine", "dot", "euclid")


def corpus(n, d, seed, kind="uniform"):
    """Uniform bytes or the quantised clustered corpus, plus a zero row, an all-255 row, exact duplicates and a sparse
    row where they fit."""
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 256, (n, d)).astype(np.uint8) if kind == "uniform" else clustered_corpus(n, d, seed)
    if n >= 8:
        x[1] = 0
        x[2] = 255
        x[4] = x[3]
        x[5] = 0
        x[5, rng.integers(0, d, max(1, d // 16))] = rng.integers(1, 256)
    return x


def queries(x, seed, B):
    rng = np.random.default_rng(seed + 1)
    d = x.shape[1]
    q = (rng.standard_normal((B, d)) * 50 + 128).astype(np.float32)
    q[0] = x[min(3, len(x) - 1)]          # a stored vector itself
    if B > 1:
        q[1] = 0.0                         # the zero query
    if B > 3:
        q[2] *= np.float32(1e-30)
        q[3] *= np.float32(1e30)
    if B > 5:
        q[4] = -q[4]
        q[5] = rng.standard_normal(d).astype(np.float32)
    return q


def check(eng, x, q, metric, what, bs, ks, filters=None, rows=None):
    """Every mode gives the same bytes, and they are the oracle's top-k."""
    want = u8_topk_many(x, q[:max(bs)], max(ks), metric, rows=rows)
    for B in bs:
        for k in ks:
            outs = []
            for mode in (0, 1, 2):
                eng.dense_set_mode(mode)
                try:
                    outs.append(eng.dense_topk(q[:B], k, filters=filters(B) if filters else None))
                finally:
                    eng.dense_set_mode(0)
            for o in outs[1:]:
                for u, v in zip(outs[0], o):
                    assert np.array_equal(u, v), f"{what} B {B} k {k}: modes differ"
            ids, sc, cnt = outs[0]
            for b in range(B):
                wi, ws = want[b][0][:k], want[b][1][:k]
                assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"{what} B {B} k {k} q {b}",
                                   mag=u8_magnitude(x, q[b], metric))


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", (1, 63, 64, 100, 1024, 4096))
def test_dimensions(engine, metric, d):
    x = corpus(3000 if d == 4096 else 8193, d, seed=d)
    q = queries(x, seed=d, B=300)
    engine.load_dense(x, metric=metric, storage="uint8")
    assert engine.dense_storage() == "uint8"
    check(engine, x, q, metric, f"{metric} d {d}", bs=(1, 17, 300), ks=(1, 100))


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("n", (1, 127, 128, 129, 8191, 20000))
def test_row_counts_batches_and_k(engine, metric, n):
    d = 100
    x = corpus(n, d, seed=n)
    q = queries(x, seed=n, B=300)
    engine.load_dense(x, metric=metric, storage="uint8")
    fb0 = engine.fallback_count()
    check(engine, x, q, metric, f"{metric} n {n}", bs=(1, 15, 16, 256, 300), ks=(1, 100, 1024))
    if n >= 8191 and metric != "euclid":   # Euclid: the 1e30 query takes K1e's fp64-resolution fallback
        assert engine.fallback_count() == fb0, "no fallbacks on a regular corpus"


@pytest.mark.parametrize("metric", METRICS)
def test_clustered_corpus(engine, metric):
    x = corpus(20000, 1024, seed=21, kind="clustered")
    q = queries(x, seed=21, B=300)
    engine.load_dense(x, metric=metric, storage="uint8")
    fb0 = engine.fallback_count()
    check(engine, x, q, metric, f"{metric} clustered", bs=(16, 300), ks=(100,))
    if metric != "euclid":
        assert engine.fallback_count() == fb0


def test_own_vector_at_distance_zero(engine):
    x = corpus(20000, 1024, seed=31)
    engine.load_dense(x, metric="euclid", storage="uint8")
    rows = np.array([0, 7, 777, 19999])
    ids, sc, _ = engine.dense_topk(x[rows].astype(np.float32), 5)
    for b, r in enumerate(rows):
        assert sc[b, 0] == 0.0 and ids[b, 0] == r


def test_u8_input_equals_float_input(built_lib):
    from sentio_b200.engine import B200Engine

    x = corpus(9000, 200, seed=41)
    q = queries(x, seed=41, B=40)
    engs = [B200Engine(0) for _ in range(3)]
    try:
        for e, v in zip(engs, (x, x.astype(np.float32), x.astype(np.float16))):
            e.load_dense(v, metric="dot", storage="uint8")
        outs = [e.dense_topk(q, 50) for e in engs]
        fetched = [e.dense_fetch(np.arange(len(x))) for e in engs]
        for o, f in zip(outs[1:], fetched[1:]):
            assert all(np.array_equal(u, v) for u, v in zip(outs[0], o))
            assert np.array_equal(fetched[0], f)
        assert np.array_equal(fetched[0], x.astype(np.float32)), "fetch returns x for every metric"
        bad = x[:2].astype(np.float32)
        bad[1, 3] = 0.5
        with pytest.raises(Exception):
            engs[0].dense_upsert([0, 1], bad)
        assert np.array_equal(engs[0].dense_fetch(np.arange(2)), x[:2].astype(np.float32))
    finally:
        for e in engs:
            e.close()


@pytest.mark.parametrize("metric", METRICS)
def test_filtered_and_grouped(engine, metric):
    n, d = 20000, 256
    x = corpus(n, d, seed=51)
    q = queries(x, seed=51, B=300)
    engine.load_dense(x, metric=metric, storage="uint8")
    rows = np.arange(n)
    engine.load_dense_tags(1, (rows % 100).astype(np.int32))              # 1 % match code 0: masked scans
    engine.load_dense_tags(2, (rows >= 1000).astype(np.int32))            # 1000 rows match code 0: gather path
    for field, match in ((1, rows[rows % 100 == 0]), (2, rows[:1000])):
        def filters(B, field=field):
            return (np.arange(B + 1, dtype=np.int32), np.full(B, field, np.int32), np.zeros(B, np.int32))
        check(engine, x, q, metric, f"{metric} filtered field {field}", bs=(3, 300), ks=(10, 100), filters=filters,
              rows=match)
    groups = (rows // 20).astype(np.int32)
    engine.load_dense_tags(3, groups)
    qg = q[:20]
    ng, codes, hits, ids, sc = engine.dense_groups(qg, 3, 10, 3)
    for b in range(len(qg)):
        want = group_search(u8_scores(x, qg[b], metric), groups.tolist(), 10, 3, ascending=metric == "euclid")
        assert int(ng[b]) == len(want), f"{metric} groups q {b}"
        for g, (code, wh) in enumerate(want):
            assert int(codes[b, g]) == code and int(hits[b, g]) == len(wh), f"{metric} group {g} q {b}"
            assert_metric_topk(ids[b, g], sc[b, g], hits[b, g], [r for r, _ in wh], [s for _, s in wh],
                               f"{metric} group {g} q {b}", mag=u8_magnitude(x, qg[b], metric))


def _same(a, b, q, what):
    n = a.dense_count[0]
    assert n == b.dense_count[0]
    assert np.array_equal(a.dense_fetch(np.arange(n)), b.dense_fetch(np.arange(n))), f"{what}: fetch"
    for B, k in ((3, 10), (300, 100)):
        for u, v in zip(a.dense_topk(q[:B], k), b.dense_topk(q[:B], k)):
            assert np.array_equal(u, v), f"{what}: B {B} k {k} differs from a fresh load"


@pytest.mark.parametrize("metric", METRICS)
def test_mutation_matches_fresh_load(built_lib, metric):
    from sentio_b200.engine import B200Engine

    mut, fresh = B200Engine(0), B200Engine(0)
    try:
        d = 100
        rng = np.random.default_rng(61)
        mirror = corpus(12000, d, seed=61)
        q = queries(mirror, seed=61, B=300)
        mut.load_dense(np.zeros((0, d), np.uint8), metric=metric, storage="uint8")
        mut.dense_reserve(5000)
        mut.dense_upsert(np.arange(len(mirror)), mirror)   # growth past the reserved capacity
        for step in range(3):
            over = rng.choice(len(mirror), 200, replace=False)
            v = corpus(200, d, seed=100 + step)
            mut.dense_upsert(over, v if step else v.astype(np.float32))
            mirror[over] = v
            app = corpus(3000, d, seed=200 + step)
            mut.dense_upsert(np.arange(len(mirror), len(mirror) + len(app)), app)
            mirror = np.concatenate([mirror, app])
            dead = rng.choice(len(mirror), 1500, replace=False)
            mf, mt = mut.dense_delete(dead)
            keep = len(mirror) - len(dead)
            m2 = mirror.copy()
            m2[mt] = m2[mf]
            mirror = m2[:keep]
        fresh.load_dense(mirror, metric=metric, storage="uint8")
        _same(mut, fresh, q, f"{metric} after mutations")
        assert np.array_equal(mut.dense_fetch(np.arange(len(mirror))), mirror.astype(np.float32))
        check(mut, mirror, q, metric, f"{metric} after mutations", bs=(17, 300), ks=(100,))
    finally:
        mut.close()
        fresh.close()


def test_duplicate_cluster_takes_the_fallback(engine):
    """3000 identical rows around the k-th best: a window wider than the winner buffer is answered by brute force, in
    the oracle's order."""
    x = corpus(20000, 256, seed=71)
    x[5000:8000] = x[5000]
    engine.load_dense(x, storage="uint8")
    rng = np.random.default_rng(72)
    q = (x[5000].astype(np.float32)[None, :] + rng.standard_normal((17, 256)).astype(np.float32)).astype(np.float32)
    fb0 = engine.fallback_count()
    ids, sc, cnt = engine.dense_topk(q, 100)
    assert engine.fallback_count() - fb0 >= len(q)
    for b in range(len(q)):
        wi, ws = u8_topk(x, q[b], 100, "cosine")
        assert ids[b].tolist() == wi.tolist()
        assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"cluster q {b}", mag=1.0)


def test_dev_entry_equals_host(engine):
    import torch

    x = corpus(20000, 1024, seed=81)
    q = queries(x, seed=81, B=64)
    engine.load_dense(x, metric="dot", storage="uint8")
    host = engine.dense_topk(q, 100)
    dev = engine.dense_topk_dev(torch.from_numpy(q).cuda(), 100)
    torch.cuda.synchronize()
    for u, v in zip(host, dev):
        assert np.array_equal(u, v.cpu().numpy())


def test_scorers_gather_x(engine):
    x = corpus(9000, 64, seed=91)
    engine.load_dense(x, storage="uint8")
    rng = np.random.default_rng(92)
    q = rng.standard_normal(64).astype(np.float32)
    ids = rng.choice(len(x), 50, replace=False)
    a = engine.semantic_mmr(q, cand_ids=ids)
    b = engine.semantic_mmr(q, cand=x[ids].astype(np.float32))
    for u, v in zip(a, b):
        assert np.array_equal(np.asarray(u), np.asarray(v))


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid"])
def test_vector_store(built_lib, dist):
    from sentio_b200.vector_store import B200VectorStore, Datatype, VectorParams

    d, metric = 64, dist.lower()
    x = corpus(3000, d, seed=95)
    s = B200VectorStore(0)
    try:
        s.create_collection("c", vectors_config=VectorParams(d, dist, datatype=Datatype.UINT8))
        s.upsert("c", [NS(id=f"p{i}", vector=x[i].tolist(), payload={"t": "a" if i % 10 == 0 else "b"})
                       for i in range(3000)])
        info = s.get_collection("c")
        assert info.config.params.vectors.datatype is Datatype.UINT8 and info.points_count == 3000
        with pytest.raises(ValueError):
            s.upsert("c", [NS(id="p1", vector=[300.0] * d, payload=None)])
        s.delete("c", [f"p{i}" for i in range(0, 3000, 7)])
        live = {f"p{i}": x[i] for i in range(3000) if i % 7}
        ids = list(live)
        X = np.stack([live[i] for i in ids])
        pos = {pid: j for j, pid in enumerate(ids)}
        rng = np.random.default_rng(96)
        Q = (rng.standard_normal((10, d)) * 40 + 128).astype(np.float32)
        flt = NS(must=[NS(key="t", match=NS(value="a"))])
        rows_a = [j for j, i in enumerate(ids) if int(i[1:]) % 10 == 0]
        for b in range(len(Q)):
            for hits, rows in ((s.search("c", Q[b], limit=10), None),
                               (s.query_points("c", query=Q[b], limit=10, query_filter=flt).points, rows_a)):
                wi, ws = u8_topk(X, Q[b], 10, metric, rows=rows)
                got = np.asarray([pos[h.id] for h in hits], np.int64)
                assert_metric_topk(got, np.asarray([h.score for h in hits]), len(hits), wi, ws, f"search {b}",
                                   mag=u8_magnitude(X, Q[b], metric))
        rec = s.retrieve("c", ["p1", "p2"], with_vectors=True)
        for r in rec:
            assert np.array_equal(np.asarray(r.vector, np.float32), live[r.id].astype(np.float32))
    finally:
        s.close()
