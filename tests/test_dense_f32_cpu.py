"""Store-level logic of float32 storage (DESIGN.md K1g) on an oracle-backed engine double (no GPU): datatype parsing
(this module's enum, qdrant_client-style enums read by ``.name``, values, plain strings, None), the float16 default
calling the engine exactly as before, FLOAT32 reaching the engine, UINT8 and float16-only engines refused by name,
``get_collection`` reporting, and rejected input leaving the collection unchanged."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from f32_oracle import f32_topk
from metric_oracle import assert_metric_topk

D = 16


class StorageOracleEngine:
    """The B200Engine calls B200VectorStore makes, answered in NumPy on the vectors as given (float32 storage).  Every
    ``load_dense`` call's keyword arguments are recorded."""

    METRICS = {"cosine": 0, "dot": 1, "euclid": 2}
    DATATYPES = {"float16": 0, "float32": 1}
    calls = []

    def __init__(self, device=0):
        self.x = np.zeros((0, D), np.float32)
        self.metric, self.storage = "cosine", "float16"
        self.dense_count, self.dense_dim = {}, {}

    def close(self):
        pass

    def load_dense(self, vecs, id_base=0, slot=0, **kw):
        StorageOracleEngine.calls.append(dict(kw))
        x = np.asarray(vecs, np.float32)
        self._validate(x)
        self.x = x.copy()
        self.metric, self.storage = kw.get("metric", "cosine"), kw.get("storage", "float16")
        self.dense_count[slot], self.dense_dim[slot] = len(x), x.shape[1]

    @staticmethod
    def _validate(x):
        if len(x) and not np.isfinite((x.astype(np.float64) ** 2).sum(1)).all():
            raise ValueError("rejected rows")

    def dense_storage(self, slot=0):
        return self.storage

    def dense_upsert(self, rows, vecs, slot=0):
        rows = np.asarray(rows, np.int64)
        v = np.asarray(vecs, np.float32)
        self._validate(v)
        x = np.concatenate([self.x, np.zeros((int((rows >= len(self.x)).sum()), D), np.float32)])
        x[rows] = v
        self.x = x
        self.dense_count[slot] = len(x)

    def dense_topk(self, q, k, slot=0, filters=None):
        assert filters is None
        q = np.atleast_2d(np.asarray(q, np.float32))
        ids = np.full((len(q), k), -1, np.int64)
        sc = np.zeros((len(q), k))
        cnt = np.zeros(len(q), np.int32)
        for b in range(len(q)):
            i, s = f32_topk(self.x, q[b], k, self.metric)
            ids[b, :len(i)], sc[b, :len(i)], cnt[b] = i, s, len(i)
        return ids, sc, cnt

    def dense_fetch(self, ids, slot=0):
        return self.x[np.asarray(ids, np.int64)]


@pytest.fixture
def store(monkeypatch):
    from sentio_b200 import vector_store

    StorageOracleEngine.calls = []
    monkeypatch.setattr(vector_store, "B200Engine", StorageOracleEngine)
    s = vector_store.B200VectorStore(0)
    yield s
    s.close()


class QdrantLikeDatatype:
    """Shaped like qdrant_client.models.Datatype members: only ``.name`` is read."""

    def __init__(self, name):
        self.name = name


@pytest.mark.parametrize("given, want", [
    (None, "FLOAT16"), ("float32", "FLOAT32"), ("Float32", "FLOAT32"), ("FLOAT16", "FLOAT16"), ("float16", "FLOAT16"),
    (QdrantLikeDatatype("FLOAT32"), "FLOAT32"), (QdrantLikeDatatype("FLOAT16"), "FLOAT16"),
])
def test_datatype_parsing_and_get_collection(store, given, want):
    from sentio_b200.vector_store import Datatype, VectorParams, parse_datatype

    assert parse_datatype(given) is Datatype[want]
    assert parse_datatype(Datatype[want]) is Datatype[want]
    assert parse_datatype(Datatype[want].value) is Datatype[want]
    store.create_collection("c", vectors_config=VectorParams(D, "Dot", datatype=given))
    info = store.get_collection("c")
    assert info.config.params.vectors.datatype is Datatype[want]
    assert info.config.params.vectors.distance.name == "DOT" and info.points_count == 0
    assert store.engine_of("c").dense_storage() == want.lower()


def test_default_path_calls_the_engine_as_before(store):
    """Without a datatype (or with FLOAT16) the engine's load_dense gets no `storage` keyword, exactly as before."""
    from sentio_b200.vector_store import Datatype, VectorParams

    store.create_collection("bulk", np.ones((3, D), np.float32))
    store.create_collection("cos", vectors_config=NS(size=D, distance="Cosine"))
    store.create_collection("dot", vectors_config=VectorParams(D, "Dot", datatype=Datatype.FLOAT16))
    store.create_collection("f32", vectors_config=VectorParams(D, "Euclid", datatype=Datatype.FLOAT32))
    assert StorageOracleEngine.calls == [{}, {}, {"metric": "dot"}, {"metric": "euclid", "storage": "float32"}]
    assert store.get_collection("bulk").config.params.vectors.datatype is Datatype.FLOAT16
    assert store.get_collection("f32").config.params.vectors.datatype is Datatype.FLOAT32


@pytest.mark.parametrize("dt", ["uint8", "UINT8", QdrantLikeDatatype("UINT8"), "int8", "bfloat16"])
def test_unsupported_datatypes_raise(store, dt):
    from sentio_b200.vector_store import VectorParams

    with pytest.raises(ValueError, match="not supported"):
        store.create_collection("u", vectors_config=VectorParams(D, "Cosine", datatype=dt))
    assert not store.collection_exists("u")
    assert StorageOracleEngine.calls == []


def test_engine_without_datatype_table_is_float16_only(monkeypatch):
    """An engine that does not list its datatypes stores float16 only: FLOAT32 is refused by name before anything is
    created; FLOAT16 and no datatype still work."""
    from sentio_b200 import vector_store

    class Float16OnlyEngine:   # METRICS but no DATATYPES table
        METRICS = StorageOracleEngine.METRICS

        def __init__(self, device=0):
            self.inner = StorageOracleEngine(device)
            self.dense_count = self.inner.dense_count

        def load_dense(self, vecs, id_base=0, slot=0, **kw):
            self.inner.load_dense(vecs, id_base, slot, **kw)

        def close(self):
            pass

    assert not hasattr(Float16OnlyEngine, "DATATYPES")
    monkeypatch.setattr(vector_store, "B200Engine", Float16OnlyEngine)
    StorageOracleEngine.calls = []
    s = vector_store.B200VectorStore(0)
    with pytest.raises(ValueError, match="float32"):
        s.create_collection("x", vectors_config=NS(size=D, distance="Cosine", datatype="float32"))
    assert not s.collection_exists("x") and StorageOracleEngine.calls == []
    s.create_collection("h", vectors_config=NS(size=D, distance="Cosine", datatype="float16"))
    s.create_collection("n", vectors_config=NS(size=D, distance="Cosine"))
    assert s.get_collection("h").config.params.vectors.datatype.name == "FLOAT16"


def test_float32_collection_end_to_end(store):
    from sentio_b200.vector_store import Datatype, VectorParams

    rng = np.random.default_rng(1)
    x = (rng.standard_normal((60, D)) * rng.uniform(0.5, 2.0, (60, 1))).astype(np.float32)
    store.create_collection("e", vectors_config=VectorParams(D, "Euclid", datatype=Datatype.FLOAT32))
    store.upsert("e", [NS(id=f"p{i}", vector=x[i].tolist(), payload={"i": i}) for i in range(60)])
    hits = store.search("e", x[7], limit=5)
    assert hits[0].id == "p7" and hits[0].score == 0.0
    wi, ws = f32_topk(x, x[7], 5, "euclid")
    assert_metric_topk(np.asarray([int(h.id[1:]) for h in hits]), np.asarray([h.score for h in hits]), 5, wi, ws)
    rec = store.retrieve("e", ["p3"], with_vectors=True)
    assert np.array_equal(np.asarray(rec[0].vector, np.float32), x[3])


def test_rejected_input_leaves_the_collection_unchanged(store):
    from sentio_b200.vector_store import VectorParams

    store.create_collection("c", vectors_config=VectorParams(D, "Cosine", datatype="float32"))
    store.upsert("c", [NS(id="a", vector=[1.0] * D, payload=None)])
    with pytest.raises(ValueError):
        store.upsert("c", [NS(id="b", vector=[np.inf] + [0.0] * (D - 1), payload=None)])
    with pytest.raises(ValueError):
        store.upsert("c", [NS(id="b", vector=[1.0] * (D - 1), payload=None)])
    info = store.get_collection("c")
    assert info.points_count == 1 and info.config.params.vectors.datatype.name == "FLOAT32"
    with pytest.raises(ValueError):
        store.create_collection("c", vectors_config=VectorParams(D, "Cosine", datatype="uint8"))
    assert store.get_collection("c").points_count == 1
    with pytest.raises(ValueError):
        store.create_collection("bad", np.full((2, D), np.nan, np.float32),
                                vectors_config=VectorParams(D, "Dot", datatype="float32"))
    assert not store.collection_exists("bad")
