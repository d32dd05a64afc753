"""Payload-filter compilation, value coding and the unsupported-filter errors of B200VectorStore.search, on an
oracle-backed engine double (no GPU)."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from oracle import dense as dense_oracle
from oracle_engine import OracleEngine
from sentio_b200 import payload_filter as pf


class FilterOracleEngine(OracleEngine):
    """OracleEngine plus the filtered-search methods of B200Engine, answered by the oracle."""

    def __init__(self, device=0):
        super().__init__()
        self.tags = {}
        self.filtered_calls = 0

    def load_dense(self, vecs, id_base=0, slot=0):
        super().load_dense(vecs, id_base, slot)
        self.tags = {}

    def load_dense_tags(self, field, codes, slot=0):
        codes = np.asarray(codes, np.int32)
        assert field < pf.MAX_TAG_FIELDS and len(codes) == len(self.rows[slot]) and codes.min(initial=0) >= -1
        self.tags[field] = codes

    def fallback_count(self):
        return 0

    def dense_topk(self, q, k, slot=0, filters=None):
        if filters is None:
            return super().dense_topk(q, k, slot)
        self.filtered_calls += 1
        off, fld, code = filters
        q = np.atleast_2d(np.asarray(q, np.float32))
        rows = self.rows[slot]
        ids = np.full((len(q), k), -1, np.int64)
        sc = np.zeros((len(q), k))
        cnt = np.zeros(len(q), np.int32)
        for b in range(len(q)):
            m = np.ones(len(rows), bool)
            for i in range(off[b], off[b + 1]):
                m &= (self.tags[int(fld[i])] == code[i]) if code[i] >= 0 else False
            idx = np.flatnonzero(m)
            if len(idx):
                i, s = dense_oracle.dense_topk(rows[idx], q[b], k)
                ids[b, :len(i)] = idx[i] + self.id_base[slot]
                sc[b, :len(i)] = s
                cnt[b] = len(i)
        return ids, sc, cnt


def _fc(key, value):
    return NS(key=key, match=NS(value=value))


@pytest.fixture
def store(monkeypatch):
    from sentio_b200 import vector_store

    monkeypatch.setattr(vector_store, "B200Engine", FilterOracleEngine)
    rng = np.random.default_rng(0)
    vecs = rng.standard_normal((300, 16)).astype(np.float32)
    payloads = []
    for i in range(300):
        md = {"source": f"s{i % 4}", "page": (True if i % 2 else 1) if i % 5 == 0 else i % 7, "flag": i % 3 == 0}
        if i % 11 == 0:
            md.pop("source")
        payloads.append({"content": f"t{i}", "metadata": md, "lang": "en" if i % 2 else "de"})
    s = vector_store.B200VectorStore(0)
    s.create_collection("c", vecs, payloads=payloads)
    return s, vecs, payloads


def test_compile_filter_shapes():
    assert pf.compile_filter(None) == []
    assert pf.compile_filter(_fc("metadata.source", "a.pdf")) == [("metadata.source", "a.pdf")]
    f = NS(must=[_fc("a", 1), _fc("b", True), _fc("c", "x")], should=None, must_not=[])
    assert pf.compile_filter(f) == [("a", 1), ("b", True), ("c", "x")]
    assert pf.compile_filter(NS(must=[])) == []
    assert pf.compile_filter(NS(must=None)) == []


def test_value_coding_keeps_types_apart():
    payloads = [{"m": {"v": True}}, {"m": {"v": 1}}, {"m": {"v": "1"}}, {"m": {}}, {"m": {"v": None}}, {"x": 1}]
    codes, table = pf.build_tag_column(payloads, "m.v")
    assert codes[3] == codes[4] == codes[5] == -1
    assert len({int(codes[0]), int(codes[1]), int(codes[2])}) == 3
    assert table[pf.value_key(True)] == codes[0] and table[pf.value_key(1)] == codes[1]
    with pytest.raises(ValueError, match="list-valued"):
        pf.build_tag_column([{"tags": ["a", "b"]}], "tags")


def test_csr_compilation_and_unknown_values():
    loaded = {}
    idx = pf.PayloadIndex([{"a": 1, "b": "x"}, {"a": 2}, {"b": "y"}], lambda f, c: loaded.__setitem__(f, c.copy()))
    off, fld, code = idx.compile([_fc("a", 2), None, NS(must=[_fc("b", "y"), _fc("a", 7)])])
    assert off.tolist() == [0, 1, 1, 3]
    assert fld.tolist() == [0, 1, 0] and code.tolist() == [1, 1, -1]
    assert loaded[0].tolist() == [0, 1, -1] and loaded[1].tolist() == [0, -1, 1]


def test_too_many_keys_raise():
    idx = pf.PayloadIndex([{f"k{i}": i for i in range(20)}], lambda f, c: None)
    for i in range(pf.MAX_TAG_FIELDS):
        idx.field(f"k{i}")
    with pytest.raises(ValueError, match="at most"):
        idx.field("k19")


def _satisfies(p, conds):
    for key, value in conds:
        v = pf.payload_value(p, key)
        if v is pf._MISSING or type(v) is not type(value) or v != value:
            return False
    return True


@pytest.mark.parametrize("conds", [
    [("metadata.source", "s1")], [("metadata.page", True)], [("metadata.page", 1)], [("metadata.flag", False)],
    [("metadata.source", "s2"), ("metadata.flag", True)], [("lang", "en")], [("metadata.source", "zzz")],
    [("source", "s1")],
])
def test_store_search_respects_filters(store, conds):
    s, vecs, payloads = store
    flt = _fc(*conds[0]) if len(conds) == 1 else NS(must=[_fc(k, v) for k, v in conds])
    want_rows = [i for i, p in enumerate(payloads) if _satisfies(p, conds)]
    q = np.random.default_rng(1).standard_normal((3, vecs.shape[1])).astype(np.float32)
    for b in range(3):
        hits = s.search("c", q[b], limit=20, query_filter=flt)
        assert all(_satisfies(h.payload, conds) for h in hits)
        assert len(hits) == min(20, len(want_rows))
    batch = s.search_batch("c", q, limit=20, query_filter=flt)
    assert [[h.id for h in r] for r in batch] == [[h.id for h in s.search("c", q[b], limit=20, query_filter=flt)]
                                                  for b in range(3)]


def test_true_and_one_are_distinct(store):
    s, vecs, payloads = store
    t = {h.id for h in s.search("c", vecs[0], limit=300, query_filter=_fc("metadata.page", True))}
    o = {h.id for h in s.search("c", vecs[0], limit=300, query_filter=_fc("metadata.page", 1))}
    assert t and o and not (t & o)
    assert all(payloads[int(i)]["metadata"]["page"] is True for i in t)


def test_no_filter_is_the_unfiltered_search(store):
    s, vecs, _ = store
    eng = s.engine_of("c")
    a = s.search("c", vecs[3], limit=10)
    b = s.search("c", vecs[3], limit=10, query_filter=None)
    c = s.search("c", vecs[3], limit=10, query_filter=NS(must=[]))
    assert [(h.id, h.score) for h in a] == [(h.id, h.score) for h in b] == [(h.id, h.score) for h in c]
    assert eng.filtered_calls == 0


def test_per_query_filter_list(store):
    s, vecs, _ = store
    flts = [None, _fc("metadata.source", "s3"), _fc("lang", "de")]
    got = s.search_batch("c", vecs[:3], limit=5, query_filter=flts)
    for b, f in enumerate(flts):
        assert [h.id for h in got[b]] == [h.id for h in s.search("c", vecs[b], limit=5, query_filter=f)]
    with pytest.raises(ValueError):
        s.search_batch("c", vecs[:3], limit=5, query_filter=flts[:2])


@pytest.mark.parametrize("flt, what", [
    (NS(must=[_fc("a", 1)], should=[_fc("a", 2)]), "should"),
    (NS(must=None, must_not=[_fc("a", 2)]), "must_not"),
    (NS(must=[NS(key="metadata.page", range=NS(gte=1), match=None)]), "range"),
    (NS(must=[NS(key="metadata.page", match=NS(any=[1, 2]))]), "any"),
    (NS(must=[NS(key="metadata.page", match=NS(text="x"))]), "text"),
    (NS(must=[NS(must=[_fc("a", 1)])]), "nested"),
    (NS(must=[_fc("metadata.page", 1.5)]), "non-scalar"),
    (NS(must=[_fc("metadata.page", [1])]), "non-scalar"),
    (NS(must=[_fc("metadata.page", {"a": 1})]), "non-scalar"),
    ({"metadata.page": 1}, "unsupported filter"),
    (NS(must=[NS(key="metadata.page")]), "no match"),
])
def test_unsupported_filters_raise(store, flt, what):
    s, vecs, _ = store
    with pytest.raises(ValueError, match=what):
        s.search("c", vecs[0], limit=5, query_filter=flt)
