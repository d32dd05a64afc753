"""Store-level logic of the Dot / Euclid distances (DESIGN.md K1e) on an oracle-backed engine double (no GPU): distance
parsing (this module's enum, qdrant_client-style enums read by ``.name``, plain strings), ``get_collection`` reporting,
Manhattan and unknown-name rejection, ascending Euclid order with distance values, and input validation."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from metric_oracle import assert_metric_topk, metric_topk, stored_metric
from oracle import dense as dense_oracle

D = 16


class MetricOracleEngine:
    """The B200Engine calls B200VectorStore makes, answered in NumPy for any metric (whole-slot reload on every write,
    which is what the device's bit-identity rule promises)."""

    METRICS = {"cosine": 0, "dot": 1, "euclid": 2}

    def __init__(self, device=0):
        self.x = np.zeros((0, D), np.float32)
        self.metric = "cosine"
        self.dense_count = {}
        self.dense_dim = {}

    def close(self):
        pass

    def load_dense(self, vecs, id_base=0, slot=0, metric="cosine"):
        if metric not in ("cosine", "dot", "euclid"):
            raise ValueError(metric)
        x = np.asarray(vecs, np.float32)
        self._validate(x, metric)
        self.x, self.metric = x.copy(), metric
        self.dense_count[slot], self.dense_dim[slot] = len(x), x.shape[1]

    @staticmethod
    def _validate(x, metric):
        if metric == "cosine" or not len(x):
            return
        ss = (x.astype(np.float64) ** 2).sum(1)
        if not np.isfinite(ss).all() or (metric == "euclid" and ss.max() > np.finfo(np.float32).max):
            raise ValueError("rejected rows")

    def dense_metric(self, slot=0):
        return self.metric

    def dense_upsert(self, rows, vecs, slot=0):
        rows = np.asarray(rows, np.int64)
        v = np.asarray(vecs, np.float32)
        self._validate(v, self.metric)
        n = len(self.x)
        x = np.concatenate([self.x, np.zeros((int((rows >= n).sum()), D), np.float32)])
        x[rows] = v
        self.x = x
        self.dense_count[slot] = len(x)

    def dense_delete(self, rows, slot=0):
        n = len(self.x)
        rows = sorted(rows)
        keep = n - len(rows)
        dead = set(rows)
        mf = np.asarray([r for r in range(keep, n) if r not in dead], np.int64)
        mt = np.asarray([r for r in rows if r < keep], np.int64)
        x = self.x.copy()
        x[mt] = x[mf]
        self.x = x[:keep]
        self.dense_count[slot] = keep
        return mf, mt

    def dense_topk(self, q, k, slot=0, filters=None):
        assert filters is None
        q = np.atleast_2d(np.asarray(q, np.float32))
        ids = np.full((len(q), k), -1, np.int64)
        sc = np.zeros((len(q), k))
        cnt = np.zeros(len(q), np.int32)
        for b in range(len(q)):
            if self.metric == "cosine":
                i, s = dense_oracle.dense_topk(dense_oracle.stored_rows(self.x), q[b], k)
            else:
                y, c = stored_metric(self.x)
                i, s = metric_topk(y, c, q[b], k, self.metric)
            ids[b, :len(i)], sc[b, :len(i)], cnt[b] = i, s, len(i)
        return ids, sc, cnt

    def dense_fetch(self, ids, slot=0):
        y, c = stored_metric(self.x)
        return (c[:, None] * y.astype(np.float64))[np.asarray(ids, np.int64)].astype(np.float32)


@pytest.fixture
def store(monkeypatch):
    from sentio_b200 import vector_store

    monkeypatch.setattr(vector_store, "B200Engine", MetricOracleEngine)
    s = vector_store.B200VectorStore(0)
    yield s
    s.close()


class QdrantLikeDistance:
    """Shaped like qdrant_client.models.Distance members: only ``.name`` is read."""

    def __init__(self, name):
        self.name = name


@pytest.mark.parametrize("given, want", [
    ("Dot", "DOT"), ("dot", "DOT"), ("DOT", "DOT"), ("Euclid", "EUCLID"), ("euclid", "EUCLID"), ("Cosine", "COSINE"),
    (QdrantLikeDistance("DOT"), "DOT"), (QdrantLikeDistance("EUCLID"), "EUCLID"), (QdrantLikeDistance("COSINE"), "COSINE"),
])
def test_distance_parsing_and_get_collection(store, given, want):
    from sentio_b200.vector_store import Distance, VectorParams, parse_distance

    assert parse_distance(given) is Distance[want]
    store.create_collection("c", vectors_config=VectorParams(D, given))
    info = store.get_collection("c")
    assert info.config.params.vectors.distance.name == want
    assert info.config.params.vectors.size == D and info.points_count == 0
    assert store.engine_of("c").dense_metric() == want.lower()


def test_empty_collections_of_every_distance(store):
    """Empty collections of every distance the engine loads; Manhattan is refused."""
    store.create_collection("c", vectors_config=NS(size=D, distance=NS(name="COSINE")))
    info = store.get_collection("c")
    assert info.points_count == 0 and info.config.params.vectors.size == D
    assert info.config.params.vectors.distance.name == "COSINE"
    assert [c.name for c in store.get_collections().collections] == ["c"]
    assert store.search("c", np.ones(D, np.float32), limit=5) == []
    with pytest.raises(ValueError):
        store.get_collection("nope")
    store.create_collection("e", vectors_config=NS(size=D, distance="Euclid"))
    assert store.get_collection("e").config.params.vectors.distance.name == "EUCLID"
    assert store.search("e", np.ones(D, np.float32), limit=5) == []
    with pytest.raises(ValueError, match="Manhattan"):
        store.create_collection("m", vectors_config=NS(size=D, distance="Manhattan"))
    store.create_collection("s", vectors_config=NS(size=D, distance="Cosine"))
    assert sorted(c.name for c in store.get_collections().collections) == ["c", "e", "s"]


def test_enum_members_and_default(store):
    from sentio_b200.vector_store import Distance

    assert (Distance.DOT.value, Distance.EUCLID.value, Distance.MANHATTAN.value) == ("Dot", "Euclid", "Manhattan")
    store.create_collection("bulk", np.ones((3, D), np.float32))   # the bulk form without vectors_config: Cosine
    assert store.get_collection("bulk").config.params.vectors.distance.name == "COSINE"


def test_engine_without_metric_table_is_cosine_only(monkeypatch):
    """An engine that does not list its metrics (the Cosine-only engine interface) gets Dot / Euclid refused by name
    before anything is created."""
    from sentio_b200 import vector_store

    class CosineOnlyEngine:   # no METRICS table, and a load_dense without `metric`
        def __init__(self, device=0):
            self.inner = MetricOracleEngine(device)
            self.dense_count = self.inner.dense_count

        def load_dense(self, vecs, id_base=0, slot=0):
            self.inner.load_dense(vecs, id_base, slot)

        def close(self):
            pass

    assert not hasattr(CosineOnlyEngine, "METRICS")
    monkeypatch.setattr(vector_store, "B200Engine", CosineOnlyEngine)
    s = vector_store.B200VectorStore(0)
    for dist in ("Dot", "Euclid"):
        with pytest.raises(ValueError, match=dist):
            s.create_collection("x", vectors_config=NS(size=D, distance=dist))
        assert not s.collection_exists("x")
    s.create_collection("c", vectors_config=NS(size=D, distance="Cosine"))
    assert s.get_collection("c").config.params.vectors.distance.name == "COSINE"


@pytest.mark.parametrize("dist", ["Manhattan", "MANHATTAN", QdrantLikeDistance("MANHATTAN"), "L1", "Hamming"])
def test_unsupported_distances_raise(store, dist):
    from sentio_b200.vector_store import VectorParams

    with pytest.raises(ValueError, match="not supported"):
        store.create_collection("m", vectors_config=VectorParams(D, dist))
    assert not store.collection_exists("m")


def test_bulk_load_with_metric(store):
    from sentio_b200.vector_store import Distance, VectorParams

    rng = np.random.default_rng(1)
    x = rng.standard_normal((50, D)).astype(np.float32) * rng.uniform(0.5, 2.0, (50, 1)).astype(np.float32)
    store.create_collection("e", x, vectors_config=VectorParams(D, Distance.EUCLID))
    q = x[7] + 0.01
    hits = store.search("e", q, limit=10)
    y, c = stored_metric(x)
    wi, ws = metric_topk(y, c, q, 10, "euclid")
    assert [h.id for h in hits] == [str(i) for i in wi]
    assert_metric_topk(np.asarray(wi), np.asarray([h.score for h in hits]), 10, wi, ws)
    assert hits[0].id == "7"
    assert all(a.score <= b.score for a, b in zip(hits, hits[1:])), "Euclid: nearest first, distance ascending"
    want = np.sqrt(((q.astype(np.float64) - c[7] * y[7].astype(np.float64)) ** 2).sum())
    assert abs(hits[0].score - want) <= 1e-12 * max(1.0, want)


def test_dot_scores_descend_and_follow_the_query_scale(store):
    from sentio_b200.vector_store import VectorParams

    rng = np.random.default_rng(2)
    x = rng.standard_normal((40, D)).astype(np.float32)
    store.create_collection("d", vectors_config=VectorParams(D, "Dot"))
    store.upsert("d", [NS(id=f"p{i}", vector=x[i].tolist(), payload={"i": i}) for i in range(40)])
    q = rng.standard_normal(D).astype(np.float32)
    a = store.search("d", q, limit=5)
    b = store.search("d", 3.0 * q, limit=5)
    assert [h.id for h in a] == [h.id for h in b]
    assert all(h1.score >= h2.score for h1, h2 in zip(a, a[1:]))
    for h1, h2 in zip(a, b):
        assert abs(h2.score - 3.0 * h1.score) <= 1e-6 * abs(h2.score)
    store.delete("d", ["p0", "p1"])
    assert store.get_collection("d").points_count == 38
    assert store.get_collection("d").config.params.vectors.distance.name == "DOT"


def test_validation_errors_leave_the_collection_unchanged(store):
    from sentio_b200.vector_store import VectorParams

    store.create_collection("e", vectors_config=VectorParams(D, "Euclid"))
    store.upsert("e", [NS(id="a", vector=[1.0] * D, payload=None)])
    with pytest.raises(ValueError):
        store.upsert("e", [NS(id="b", vector=[np.inf] + [0.0] * (D - 1), payload=None)])
    with pytest.raises(ValueError):   # ||x||^2 = 16 * 1e38^2 is past the fp32 range
        store.upsert("e", [NS(id="b", vector=[1e38] * D, payload=None)])
    assert store.get_collection("e").points_count == 1
    with pytest.raises(ValueError):
        store.create_collection("bad", np.full((2, D), 1e38, np.float32), vectors_config=VectorParams(D, "Euclid"))
    assert not store.collection_exists("bad")
