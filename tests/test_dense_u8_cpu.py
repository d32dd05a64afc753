"""Store-level logic of uint8 storage (DESIGN.md K1i) on an oracle-backed engine double (no GPU): datatype parsing and
``get_collection``, uint8 and float input reaching the engine as the same bytes, refused input (fractional, negative,
256, NaN, wrong dimension) leaving the collection unchanged, engines that do not list uint8 refusing it, the query
column permutation of the uint8 scan, and the uint8 oracle against a row-by-row brute force."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from metric_oracle import assert_metric_topk
from u8_oracle import clustered_corpus, u8_brute_topk, u8_query_column, u8_topk, u8_topk_many

D = 16


class U8OracleEngine:
    """The B200Engine calls B200VectorStore makes, answered in NumPy on the stored uint8 rows.  Every ``load_dense`` /
    ``dense_upsert`` call's arguments are recorded."""

    METRICS = {"cosine": 0, "dot": 1, "euclid": 2}
    DATATYPES = {"float16": 0, "float32": 1, "uint8": 2}
    calls = []

    def __init__(self, device=0):
        self.x = np.zeros((0, D), np.uint8)
        self.metric, self.storage = "cosine", "float16"
        self.dense_count, self.dense_dim = {}, {}

    def close(self):
        pass

    def load_dense(self, vecs, id_base=0, slot=0, **kw):
        U8OracleEngine.calls.append(("load", np.asarray(vecs).copy(), dict(kw)))
        v = np.asarray(vecs)
        assert kw.get("storage") == "uint8" and v.dtype == np.uint8, "a uint8 collection passes uint8 rows"
        self.x = v.copy()
        self.metric, self.storage = kw.get("metric", "cosine"), "uint8"
        self.dense_count[slot], self.dense_dim[slot] = len(v), v.shape[1]

    def dense_storage(self, slot=0):
        return self.storage

    def dense_upsert(self, rows, vecs, slot=0):
        v = np.asarray(vecs)
        U8OracleEngine.calls.append(("upsert", v.copy(), {}))
        assert v.dtype == np.uint8
        rows = np.asarray(rows, np.int64)
        x = np.concatenate([self.x, np.zeros((int((rows >= len(self.x)).sum()), D), np.uint8)])
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
            i, s = u8_topk(self.x, q[b], k, self.metric)
            ids[b, :len(i)], sc[b, :len(i)], cnt[b] = i, s, len(i)
        return ids, sc, cnt

    def dense_fetch(self, ids, slot=0):
        return self.x[np.asarray(ids, np.int64)].astype(np.float32)


@pytest.fixture
def store(monkeypatch):
    from sentio_b200 import vector_store

    U8OracleEngine.calls = []
    monkeypatch.setattr(vector_store, "B200Engine", U8OracleEngine)
    s = vector_store.B200VectorStore(0)
    yield s
    s.close()


class QdrantLikeDatatype:
    def __init__(self, name):
        self.name = name


@pytest.mark.parametrize("dt", ["uint8", "UINT8", "Uint8", QdrantLikeDatatype("UINT8")])
def test_uint8_parses_and_is_reported(store, dt):
    from sentio_b200.vector_store import Datatype, VectorParams, parse_datatype

    assert parse_datatype(dt) is Datatype.UINT8
    store.create_collection("u", vectors_config=VectorParams(D, "Dot", datatype=dt))
    assert store.get_collection("u").config.params.vectors.datatype is Datatype.UINT8
    kind, v, kw = U8OracleEngine.calls[0]
    assert kind == "load" and kw == {"metric": "dot", "storage": "uint8"} and v.shape == (0, D)


@pytest.mark.parametrize("dt", ["int8", "bfloat16", QdrantLikeDatatype("INT8")])
def test_other_datatypes_still_refused(dt):
    from sentio_b200.vector_store import parse_datatype

    with pytest.raises(ValueError, match="not supported"):
        parse_datatype(dt)


def test_uint8_and_float_input_reach_the_engine_identically(store):
    from sentio_b200.vector_store import VectorParams

    rng = np.random.default_rng(3)
    x = rng.integers(0, 256, (40, D)).astype(np.uint8)
    store.create_collection("a", x, vectors_config=VectorParams(D, "Euclid", datatype="uint8"))
    store.create_collection("b", x.astype(np.float32), vectors_config=VectorParams(D, "Euclid", datatype="uint8"))
    store.create_collection("c", x.astype(np.float16), vectors_config=VectorParams(D, "Euclid", datatype="uint8"))
    loads = [c for c in U8OracleEngine.calls if c[0] == "load"]
    assert all(v.dtype == np.uint8 and np.array_equal(v, x) for _, v, _ in loads)
    store.create_collection("e", vectors_config=VectorParams(D, "Euclid", datatype="uint8"))
    store.upsert("e", [NS(id=i, vector=x[i].tolist(), payload=None) for i in range(40)])
    ups = [c for c in U8OracleEngine.calls if c[0] == "upsert"]
    assert np.array_equal(ups[-1][1], x)
    hits = store.search("e", x[7].astype(np.float32), limit=5)
    assert hits[0].id == 7 and hits[0].score == 0.0
    rec = store.retrieve("e", [3], with_vectors=True)
    assert np.array_equal(np.asarray(rec[0].vector, np.float32), x[3].astype(np.float32))


@pytest.mark.parametrize("bad", [0.5, -1.0, 256.0, float("nan"), float("inf"), -0.25, 255.5])
def test_refused_values_leave_the_collection_unchanged(store, bad):
    from sentio_b200.vector_store import VectorParams

    store.create_collection("c", vectors_config=VectorParams(D, "Cosine", datatype="uint8"))
    store.upsert("c", [NS(id="a", vector=[1.0] * D, payload=None)])
    n_calls = len(U8OracleEngine.calls)
    with pytest.raises(ValueError):
        store.upsert("c", [NS(id="b", vector=[bad] + [0.0] * (D - 1), payload=None)])
    with pytest.raises(ValueError):
        store.upsert("c", [NS(id="a", vector=[2.0] * (D - 1), payload=None)])   # wrong dimension
    assert len(U8OracleEngine.calls) == n_calls
    info = store.get_collection("c")
    assert info.points_count == 1 and info.config.params.vectors.datatype.name == "UINT8"
    with pytest.raises(ValueError):
        store.create_collection("bad", np.full((2, D), bad, np.float32),
                                vectors_config=VectorParams(D, "Dot", datatype="uint8"))
    assert not store.collection_exists("bad")


def test_engines_without_uint8_refuse_it(monkeypatch):
    from sentio_b200 import vector_store

    class NoU8Engine(U8OracleEngine):
        DATATYPES = {"float16": 0, "float32": 1}

    monkeypatch.setattr(vector_store, "B200Engine", NoU8Engine)
    U8OracleEngine.calls = []
    s = vector_store.B200VectorStore(0)
    with pytest.raises(ValueError, match="not supported"):
        s.create_collection("x", vectors_config=NS(size=D, distance="Cosine", datatype="uint8"))
    assert not s.collection_exists("x") and U8OracleEngine.calls == []


def test_engine_table_lists_uint8():
    from sentio_b200.engine import B200Engine

    assert B200Engine.DATATYPES["uint8"] == 2


def test_query_column_permutation():
    """A bijection on every 64-column block, and the permuted dot product equals the natural one (to fp32 summation
    order; exactly in fp64 on integer data)."""
    perm = [u8_query_column(c) for c in range(64)]
    assert sorted(perm) == list(range(64))
    # thread t (lane % 4) supplies, for k16 step s, the A columns 2t, 2t + 1, 2t + 8, 2t + 9 from its bytes 16t + 4s + j
    for t in range(4):
        for s in range(4):
            got = [perm[16 * t + 4 * s + j] - 16 * s for j in range(4)]
            assert got == [2 * t, 2 * t + 1, 2 * t + 8, 2 * t + 9]
    rng = np.random.default_rng(5)
    d = 192
    x = rng.integers(0, 256, d).astype(np.float64)
    q = rng.integers(-1000, 1000, d).astype(np.float64)
    qp = np.zeros(d)
    for c in range(d):
        qp[(c & ~63) + u8_query_column(c & 63)] = q[c]
    # the kernel's A operand at permuted column p holds the byte at natural column c: a_perm[perm(c)] = x[c]
    xp = np.zeros(d)
    for c in range(d):
        xp[(c & ~63) + u8_query_column(c & 63)] = x[c]
    assert float(xp @ qp) == float(x @ q)


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclid"])
def test_oracle_matches_brute_force(metric):
    rng = np.random.default_rng(7)
    x = np.concatenate([rng.integers(0, 256, (50, 10)), np.zeros((2, 10)), np.full((2, 10), 255),
                        clustered_corpus(30, 10, seed=8)]).astype(np.uint8)
    x[60] = x[3]
    qs = [rng.standard_normal(10).astype(np.float32) * s for s in (1e-3, 1.0, 1e3)]
    qs += [x[3].astype(np.float32), np.zeros(10, np.float32)]
    many = u8_topk_many(x, np.stack(qs), 20, metric)
    for b, q in enumerate(qs):
        wi, ws = u8_brute_topk(x, q, 20, metric)
        gi, gs = u8_topk(x, q, 20, metric)
        assert_metric_topk(gi, gs, len(gi), wi, ws, f"{metric} q {b}", mag=1.0 if metric == "cosine" else None)
        assert np.array_equal(gi, many[b][0])
