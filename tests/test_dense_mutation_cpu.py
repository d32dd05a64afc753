"""B200VectorStore writes (upsert / delete / get_collection / retrieve) on an oracle-backed engine double that
implements the documented swap-compaction plan in NumPy (no GPU): id / payload / row bookkeeping, last-wins
duplicates, ignored unknown deletes, every ValueError leaving the collection unchanged, payload-index updates, and
searches racing mutations from other threads."""
import threading
import time
from types import SimpleNamespace as NS

import numpy as np
import pytest

from oracle import dense as dense_oracle
from oracle_engine import OracleEngine
from sentio_b200 import payload_filter as pf

D = 16


def compaction_plan(n, rows):
    """The documented rule: the surviving rows among the last |D| rows, ascending, fill the deleted rows below
    n - |D|, ascending."""
    rows = sorted(rows)
    keep = n - len(rows)
    holes = [r for r in rows if r < keep]
    dead = set(rows)
    src = [r for r in range(keep, n) if r not in dead]
    assert len(src) == len(holes)
    return np.asarray(src, np.int64), np.asarray(holes, np.int64)


class MutableOracleEngine(OracleEngine):
    """OracleEngine plus filtered search and the mutation methods of B200Engine, answered in NumPy."""

    def __init__(self, device=0):
        super().__init__()
        self.tags = {}
        self.dense_count = {}

    def load_dense(self, vecs, id_base=0, slot=0):
        super().load_dense(vecs, id_base, slot)
        self.tags = {}
        self.dense_count[slot] = len(self.rows[slot])

    def load_dense_tags(self, field, codes, slot=0):
        codes = np.asarray(codes, np.int32)
        assert field < pf.MAX_TAG_FIELDS and len(codes) == len(self.rows[slot]) and codes.min(initial=0) >= -1
        self.tags[field] = codes.copy()

    def fallback_count(self):
        return 0

    def dense_reserve(self, n_cap, slot=0):
        pass

    def dense_upsert(self, rows, vecs, slot=0):
        rows = np.asarray(rows, np.int64)
        n = len(self.rows[slot])
        app = np.sort(rows[rows >= n])
        assert len(set(rows.tolist())) == len(rows) and np.array_equal(app, np.arange(n, n + len(app)))
        x = np.concatenate([self.rows[slot], np.zeros((len(app), self.dense_dim[slot]), np.float16)])
        x[rows] = dense_oracle.stored_rows(np.asarray(vecs, np.float32))
        self.rows[slot] = x
        for f in self.tags:
            self.tags[f] = np.concatenate([self.tags[f], np.full(len(app), -1, np.int32)])
            self.tags[f][rows] = -1
        self.dense_count[slot] = len(x)

    def dense_tags_write(self, field, rows, codes, slot=0):
        assert np.all(np.asarray(codes) >= -1)
        self.tags[field][np.asarray(rows, np.int64)] = codes

    def dense_delete(self, rows, slot=0):
        n = len(self.rows[slot])
        mf, mt = compaction_plan(n, list(rows))
        keep = n - len(rows)
        x = self.rows[slot].copy()
        x[mt] = x[mf]
        self.rows[slot] = x[:keep]
        for f in self.tags:
            t = self.tags[f].copy()
            t[mt] = t[mf]
            self.tags[f] = t[:keep]
        self.dense_count[slot] = keep
        return mf, mt

    def dense_topk(self, q, k, slot=0, filters=None):
        if filters is None:
            return super().dense_topk(q, k, slot)
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
                ids[b, :len(i)] = idx[i]
                sc[b, :len(i)] = s
                cnt[b] = len(i)
        return ids, sc, cnt

    def dense_fetch(self, ids, slot=0):
        return self.rows[slot][np.asarray(ids, np.int64)].astype(np.float32)

    def semantic_mmr(self, q, cand=None, cand_ids=None, **kw):
        time.sleep(0.001)   # a ctypes call releases the GIL: other threads run between the caller's lookup and the gather
        return super().semantic_mmr(q, cand=cand, cand_ids=cand_ids, **kw)


def _fc(key, value):
    return NS(key=key, match=NS(value=value))


def _pt(pid, vec, payload=None):
    return NS(id=pid, vector=vec, payload=payload)


@pytest.fixture
def vs(monkeypatch):
    from sentio_b200 import vector_store

    monkeypatch.setattr(vector_store, "B200Engine", MutableOracleEngine)
    s = vector_store.B200VectorStore(0)
    s.create_collection("c", vectors_config=NS(size=D, distance=NS(name="COSINE")))
    return s


def _vec(rng, n):
    return rng.standard_normal((n, D)).astype(np.float32)


def _content(s, name="c"):
    """{id: (stored row, payload)} through the public API plus the internal invariants."""
    col = s._collections[name]
    eng = col.engine
    assert len(col.ids) == len(col.payloads) == len(eng.rows[0]) == eng.dense_count[0]
    assert col.row_of == {pid: i for i, pid in enumerate(col.ids)}
    return {pid: (eng.rows[0][i].tobytes(), col.payloads[i]) for i, pid in enumerate(col.ids)}


def _expected_search(model, q, k, conds=()):
    """Oracle answer over a {id: (vec32, payload)} model: (ids, scores) best first; ties by the store's row order are
    not checked here (distinct random vectors)."""
    ids = [pid for pid, (_v, p) in model.items() if all(pf.payload_value(p, key) == val and
                                                        type(pf.payload_value(p, key)) is type(val)
                                                        for key, val in conds)]
    if not ids:
        return [], []
    x = dense_oracle.stored_rows(np.stack([model[i][0] for i in ids]))
    i, sc = dense_oracle.dense_topk(x, q, k)
    return [ids[j] for j in i], list(sc)


def test_empty_collection_and_info(vs):
    info = vs.get_collection("c")
    assert info.points_count == 0 and info.config.params.vectors.size == D
    assert info.config.params.vectors.distance.name == "COSINE"
    assert [c.name for c in vs.get_collections().collections] == ["c"]
    assert vs.search("c", np.ones(D, np.float32), limit=5) == []
    with pytest.raises(ValueError):
        vs.get_collection("nope")
    with pytest.raises(ValueError, match="Euclid"):
        vs.create_collection("e", vectors_config=NS(size=D, distance="Euclid"))
    vs.create_collection("s", vectors_config=NS(size=D, distance="Cosine"))
    assert sorted(c.name for c in vs.get_collections().collections) == ["c", "s"]


def test_upsert_overwrite_delete_bookkeeping(vs):
    rng = np.random.default_rng(0)
    model = {}
    v = _vec(rng, 40)
    r = vs.upsert("c", [_pt(str(i), v[i].tolist(), {"content": f"t{i}", "metadata": {"s": i % 3}}) for i in range(40)])
    assert r.status == "completed"
    model.update({str(i): (v[i], {"content": f"t{i}", "metadata": {"s": i % 3}}) for i in range(40)})
    # re-ingest of ids "0".."9" overwrites in place; "40".."44" append (Batch form)
    w = _vec(rng, 15)
    ids = [str(i) for i in range(10)] + [str(i) for i in range(40, 45)]
    vs.upsert("c", NS(ids=ids, vectors=w, payloads=[{"content": f"u{i}"} for i in ids]))
    model.update({pid: (w[j], {"content": f"u{pid}"}) for j, pid in enumerate(ids)})
    assert vs.get_collection("c").points_count == 45
    assert vs.rows_of("c", ["0", "44"]).tolist() == [0, 44]
    vs.delete("c", NS(points=["3", "44", "7", "nope", "20"]))
    for pid in ("3", "44", "7", "20"):
        model.pop(pid)
    vs.delete("c", ["39", "39", "unknown"])
    model.pop("39")
    got = _content(vs)
    assert set(got) == set(model)
    for pid, (vec, payload) in model.items():
        assert got[pid][0] == dense_oracle.stored_rows(vec[None]).tobytes() and got[pid][1] == payload
    recs = vs.retrieve("c", ["0", "nope", "21"], with_vectors=True)
    assert [rc.id for rc in recs] == ["0", "21"]
    assert np.array_equal(np.float32(recs[0].vector), dense_oracle.stored_rows(model["0"][0][None])[0].astype(np.float32))
    q = _vec(rng, 4)
    for b in range(4):
        want, ws = _expected_search(model, q[b], 10)
        hits = vs.search("c", q[b], limit=10)
        assert [h.id for h in hits] == want and np.allclose([h.score for h in hits], ws)
    recs, nxt = vs.scroll("c", limit=100)
    assert nxt is None and {rc.id for rc in recs} == set(model)


def test_last_occurrence_wins(vs):
    rng = np.random.default_rng(1)
    v = _vec(rng, 3)
    vs.upsert("c", [_pt("a", v[0], {"k": 1}), _pt("b", v[1], {"k": 2}), _pt("a", v[2], {"k": 3})])
    got = _content(vs)
    assert list(got) == ["a", "b"]
    assert got["a"] == (dense_oracle.stored_rows(v[2][None]).tobytes(), {"k": 3})


def test_delete_plan_follows_the_rule(vs):
    rng = np.random.default_rng(2)
    vs.upsert("c", [_pt(str(i), v) for i, v in enumerate(_vec(rng, 20))])
    eng = vs.engine_of("c")
    before = list(vs._collections["c"].ids)
    vs.delete("c", ["2", "5", "18", "19", "17"])       # holes 2, 5; tail 15..19 with 17, 18, 19 deleted
    ids = vs._collections["c"].ids
    assert ids[2] == "15" and ids[5] == "16" and len(ids) == 15
    assert [i for i in before if i not in {"2", "5", "17", "18", "19"}] == sorted(ids, key=int)
    assert eng.dense_count[0] == 15
    vs.delete("c", [str(i) for i in range(20)])
    assert vs.get_collection("c").points_count == 0 and vs.search("c", np.ones(D), limit=3) == []
    vs.upsert("c", [_pt("z", np.ones(D))])
    assert [h.id for h in vs.search("c", np.ones(D), limit=3)] == ["z"]


def _snapshot(vs, flt_key="metadata.s"):
    col = vs._collections["c"]
    pi = col._payload_index
    return (_content(vs), {k: (f, dict(t)) for k, (f, t) in pi.fields.items()} if pi else None,
            {f: c.copy() for f, c in col.engine.tags.items()})


@pytest.mark.parametrize("bad, what", [
    ([_pt("x", np.ones(D + 1))], "dimension"),
    ([_pt("x", [np.nan] + [1.0] * (D - 1))], "NaN"),
    ([_pt("x", [np.inf] * D)], "NaN"),
    ([_pt("x", {"text": np.ones(D)})], "named vectors"),
    (NS(ids=["x"], vectors={"text": [np.ones(D)]}, payloads=None), "named vectors"),
    ([_pt("0", np.ones(D), {"metadata": {"s": [1, 2]}})], "list-valued"),
    ([_pt("new", np.ones(D), {"metadata": {"s": {"a": 1}}})], "list-valued"),
    ([_pt("0", np.ones(D)), _pt("y", np.ones(D + 2))], "dimension"),
])
def test_rejected_upserts_leave_the_collection_unchanged(vs, bad, what):
    rng = np.random.default_rng(3)
    vs.upsert("c", [_pt(str(i), v, {"metadata": {"s": i % 3}}) for i, v in enumerate(_vec(rng, 12))])
    flt = _fc("metadata.s", 1)
    q = _vec(rng, 1)[0]
    vs.search("c", q, limit=5, query_filter=flt)     # indexes metadata.s
    before = _snapshot(vs)
    res = [(h.id, h.score) for h in vs.search("c", q, limit=5, query_filter=flt)]
    with pytest.raises(ValueError, match=what):
        vs.upsert("c", bad)
    after = _snapshot(vs)
    assert after[0] == before[0] and after[1] == before[1]
    assert all(np.array_equal(after[2][f], before[2][f]) for f in before[2])
    assert vs.get_collection("c").points_count == 12
    assert [(h.id, h.score) for h in vs.search("c", q, limit=5, query_filter=flt)] == res


def test_filter_delete_and_create_errors(vs):
    with pytest.raises(ValueError, match="deleting by filter"):
        vs.delete("c", NS(filter=NS(must=[_fc("a", 1)])))
    with pytest.raises(ValueError):
        vs.create_collection("e")
    assert vs.get_collection("c").points_count == 0


def test_payload_index_updates(vs):
    rng = np.random.default_rng(4)
    v = _vec(rng, 30)
    vs.upsert("c", [_pt(str(i), v[i], {"metadata": {"s": f"v{i % 2}"}}) for i in range(30)])
    q = _vec(rng, 1)[0]
    assert {h.payload["metadata"]["s"] for h in vs.search("c", q, limit=30, query_filter=_fc("metadata.s", "v0"))} == {"v0"}
    # new values for an indexed key get new codes; an overwrite without the key reads -1
    vs.upsert("c", [_pt("0", v[0], {"metadata": {"s": "new"}}), _pt("1", v[1], {}), _pt("30", v[2], {"metadata": {"s": "new"}})])
    hits = vs.search("c", q, limit=30, query_filter=_fc("metadata.s", "new"))
    assert sorted(h.id for h in hits) == ["0", "30"]
    assert "1" not in {h.id for h in vs.search("c", q, limit=30, query_filter=_fc("metadata.s", "v1"))}
    # codes travel with their rows through a delete
    vs.delete("c", ["2", "4", "6"])
    model = {pid: (None, p) for pid, p in zip(vs._collections["c"].ids, vs._collections["c"].payloads)}
    for val in ("v0", "v1", "new"):
        want = {pid for pid, (_v, p) in model.items() if p.get("metadata", {}).get("s") == val}
        assert {h.id for h in vs.search("c", q, limit=40, query_filter=_fc("metadata.s", val))} == want
    # a key indexed later is built from the current payloads
    vs.upsert("c", [_pt("7", v[7], {"lang": "de"})])
    assert [h.id for h in vs.search("c", q, limit=40, query_filter=_fc("lang", "de"))] == ["7"]
    codes, added = pf.build_tag_column([{"k": "a"}, {"k": "b"}, {}], "k", {pf.value_key("a"): 0})
    assert codes.tolist() == [0, 1, -1] and added == {pf.value_key("b"): 1}


def test_searches_racing_mutations_see_a_snapshot(vs):
    rng = np.random.default_rng(5)
    pool = _vec(rng, 400)
    q = _vec(rng, 3)
    snapshots = []

    def snap():
        col = vs._collections["c"]
        model = {pid: (pool[int(pid)], p) for pid, p in zip(col.ids, col.payloads)}
        snapshots.append([tuple(_expected_search(model, q[b], 5)[0]) for b in range(3)])

    vs.upsert("c", [_pt(str(i), pool[i]) for i in range(100)])
    snap()
    answers, errors = [], []
    stop = threading.Event()

    def searcher():
        try:
            while not stop.is_set():
                res = vs.search_batch("c", q, limit=5)
                answers.append([tuple(h.id for h in r) for r in res])
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)

    threads = [threading.Thread(target=searcher) for _ in range(3)]
    for t in threads:
        t.start()
    for step in range(30):
        if step % 3 == 2:
            ids = [str(i) for i in rng.choice(400, 15, replace=False)]
            vs.delete("c", ids)
        else:
            ids = rng.choice(400, 20, replace=False)
            vs.upsert("c", [_pt(str(i), pool[i]) for i in ids])
        snap()
    stop.set()
    for t in threads:
        t.join()
    assert not errors and answers
    allowed = {tuple(s) for s in snapshots}
    assert all(tuple(a) in allowed for a in answers)


def test_bare_filter_and_other_selectors_raise(vs):
    rng = np.random.default_rng(6)
    vs.upsert("c", [_pt(str(i), v, {"k": i}) for i, v in enumerate(_vec(rng, 5))])
    before = _content(vs)
    for sel in (NS(must=[_fc("k", 1)]), NS(filter=NS(must=[_fc("k", 1)])), "0", {"points": ["0"]}):
        with pytest.raises(ValueError, match="not supported"):
            vs.delete("c", sel)
    assert _content(vs) == before
    vs.delete("c", ("0", "1"))
    assert vs.get_collection("c").points_count == 3


def test_gpu_scorers_racing_mutations_score_their_own_points(vs):
    """SemanticSimilarityScorer / MMRScorer gather candidate vectors by id from the store: the id -> row lookup and the
    device call must not straddle an upsert / delete that moves rows."""
    from sentio_b200.document import Document
    from sentio_b200.retrievers.scorers import MMRScorer, SemanticSimilarityScorer

    rng = np.random.default_rng(7)
    pool = _vec(rng, 200)
    vs.upsert("c", [_pt(str(i), pool[i]) for i in range(200)])
    qv = _vec(rng, 1)[0]

    def no_text_embedding(texts):
        raise AssertionError("candidates must come from the store")

    emb = NS(embed_sync=lambda t: qv, embed_many_sync=no_text_embedding)
    scored = [str(i) for i in range(185, 200)]   # the tail: the first deletes move these rows
    docs = [Document(text="x", id=i) for i in scored]
    scorers = [SemanticSimilarityScorer(emb, vector_source=(vs, "c")), MMRScorer(emb, vector_source=(vs, "c"))]
    want = [s.score("q", docs) for s in scorers]
    assert all(any(x != 0.0 for x in w) for w in want)
    bad, stop = [], threading.Event()

    def worker(j):
        while not stop.is_set():
            got = scorers[j].score("q", docs)
            if got != want[j]:
                bad.append(got)

    threads = [threading.Thread(target=worker, args=(j,)) for j in (0, 1, 0)]
    for t in threads:
        t.start()
    others = [str(i) for i in range(185)]
    for _ in range(40):
        gone = [others[i] for i in rng.choice(len(others), 20, replace=False)]
        vs.delete("c", gone)
        vs.upsert("c", [_pt(i, pool[int(i)]) for i in gone])
    stop.set()
    for t in threads:
        t.join()
    assert not bad
    assert set(vs.rows_of("c", scored).tolist()) != set(range(185, 200))   # the scored points did move
