"""Dense slot mutation on the device (sb_dense_upsert / sb_dense_tags_write / sb_dense_delete / sb_dense_reserve): after
every step of seeded mutation sequences the slot must equal, bit for bit, a slot freshly loaded with the same rows in
the same order (stored rows, search results of both scans, filtered search), the delete plan must follow the documented
rule, and results must match the fp64 oracle.  Plus the stale-tensor-map case, growth with and without reserve, the
vector store end to end, and a search in flight on a side stream while a delete runs."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from helpers import assert_topk_matches
from oracle import dense as dense_oracle

pytestmark = pytest.mark.gpu

BS = (1, 5, 16, 256, 260)
KS = (1, 10, 100)
ZERO_Q = 4   # in the zero-query batch, query 4 is all zeros: the first k rows, score 0


def compaction_plan(n, rows):
    rows = sorted(rows)
    keep = n - len(rows)
    dead = set(rows)
    return (np.asarray([r for r in range(keep, n) if r not in dead], np.int64),
            np.asarray([r for r in rows if r < keep], np.int64))


@pytest.fixture(scope="module")
def engines(built_lib):
    from sentio_b200.engine import B200Engine

    a, b = B200Engine(0), B200Engine(0)
    yield a, b
    a.close()
    b.close()


def _oracle_top(x16, q, kmax=100):
    x = x16.astype(np.float64)
    q64 = q.astype(np.float64)
    den = np.sqrt((x * x).sum(1))[:, None] * np.sqrt((q64 * q64).sum(1))[None, :]
    s = np.zeros((len(x), len(q)))
    np.divide(x @ q64.T, den, out=s, where=den > 0)
    idx = np.arange(len(x))
    out = []
    for b in range(len(q)):
        o = np.lexsort((idx, -s[:, b]))[:kmax]
        out.append((o, s[o, b]))
    return out


def _search(eng, q, k, mode, filters=None):
    eng.dense_set_mode(mode)
    try:
        return eng.dense_topk(q, k, filters=filters) if filters is not None else eng.dense_topk(q, k)
    finally:
        eng.dense_set_mode(0)


def _check_state(mut, fresh, mirror, q, what, tags=None, conds=None):
    """mirror: fp32 input rows in row order; tags: {field: codes}; conds: per-query filter (CSR) or None."""
    n = len(mirror)
    fresh.load_dense(mirror)
    if tags is not None:
        for f, c in tags.items():
            fresh.load_dense_tags(f, c)
    assert mut.dense_count[0] == n
    stored = dense_oracle.stored_rows(mirror)
    if n:
        got = mut.dense_fetch(np.arange(n))
        assert np.array_equal(got, fresh.dense_fetch(np.arange(n))), f"{what}: stored rows differ from a fresh load"
        assert np.all(np.abs(got.astype(np.float16).view(np.int16).astype(np.int32)
                             - stored.view(np.int16).astype(np.int32)) <= 1), f"{what}: rows vs oracle"
    top = _oracle_top(stored, q) if conds is None else None
    for mode in (1, 2):
        for B in BS:
            for k in KS:
                filt = None if conds is None else conds(B)
                a = _search(mut, q[:B], k, mode, filt)
                b = _search(fresh, q[:B], k, mode, filt)
                for x, y in zip(a, b):
                    assert np.array_equal(x, y), f"{what}: mode {mode} B {B} k {k} differs from a fresh load"
                if top is None:
                    continue
                ids, sc, cnt = a
                for j in range(B):
                    wi, ws = top[j][0][:k], top[j][1][:k]
                    assert_topk_matches(ids[j], sc[j], cnt[j], wi, ws, what=f"{what} mode {mode} B {B} k {k} q {j}")
    if conds is not None:
        return 0
    # the all-zero query ties every row, so its whole candidate list lies in the error window and the merge hands it
    # to the brute-force kernel by design: checked in batches of its own, whose fallbacks the caller discounts
    fb = mut.fallback_count()
    qz = q[:16].copy()
    qz[ZERO_Q] = 0.0
    for mode in (1, 2):
        for k in KS:
            ids, sc, cnt = _search(mut, qz, k, mode)
            for x, y in zip((ids, sc, cnt), _search(fresh, qz, k, mode)):
                assert np.array_equal(x, y), f"{what}: zero-query batch mode {mode} k {k} differs from a fresh load"
            assert ids[ZERO_Q, :min(k, n)].tolist() == list(range(min(k, n)))
            assert cnt[ZERO_Q] == min(k, n) and np.all(sc[ZERO_Q, :min(k, n)] == 0.0)
    return mut.fallback_count() - fb


def _queries(rng, d):
    return rng.standard_normal((max(BS), d)).astype(np.float32)


@pytest.mark.parametrize("d, n0", [(256, 20000), (1024, 12000)])
def test_random_mutation_sequence_matches_fresh_load(engines, d, n0):
    mut, fresh = engines
    rng = np.random.default_rng(d)
    mirror = rng.standard_normal((n0, d)).astype(np.float32)
    mut.load_dense(mirror)
    q = _queries(rng, d)
    q[2] = mirror[77]
    fb0 = mut.fallback_count()

    def upsert(rows, vecs):
        nonlocal mirror
        rows = np.asarray(rows, np.int64)
        app = int((rows >= len(mirror)).sum())
        mirror = np.concatenate([mirror, np.zeros((app, d), np.float32)])
        mirror[rows] = vecs
        mut.dense_upsert(rows, vecs)

    def append(m, shuffle=True):
        rows = np.arange(len(mirror), len(mirror) + m)
        if shuffle:
            rng.shuffle(rows)
        upsert(rows, rng.standard_normal((m, d)).astype(np.float32))

    def delete(rows):
        nonlocal mirror
        rows = np.asarray(rows, np.int64)
        mf, mt = mut.dense_delete(rows)
        wf, wt = compaction_plan(len(mirror), rows.tolist())
        assert np.array_equal(mf, wf) and np.array_equal(mt, wt), "delete plan does not follow the documented rule"
        mirror[mt] = mirror[mf]
        mirror = mirror[:len(mirror) - len(rows)]

    steps = [
        ("append 1", lambda: append(1)),
        ("append 7", lambda: append(7)),
        ("append 300", lambda: append(300)),
        ("append 5000", lambda: append(5000)),
        ("overwrite 500", lambda: upsert(rng.choice(len(mirror), 500, replace=False),
                                         rng.standard_normal((500, d)).astype(np.float32))),
        ("overwrite + append", lambda: upsert(rng.permutation(np.r_[rng.choice(len(mirror), 50, replace=False),
                                                                    np.arange(len(mirror), len(mirror) + 40)]),
                                              rng.standard_normal((90, d)).astype(np.float32))),
        ("delete holes", lambda: delete(rng.choice(len(mirror) - 2000, 200, replace=False))),
        ("delete tail", lambda: delete(np.arange(len(mirror) - 150, len(mirror)))),
        ("delete both", lambda: delete(np.r_[rng.choice(len(mirror) - 400, 150, replace=False),
                                             len(mirror) - 1 - rng.choice(400, 150, replace=False)])),
        ("below wgmma threshold", lambda: delete(rng.choice(len(mirror), len(mirror) - 8000, replace=False))),
        ("above wgmma threshold", lambda: append(300)),
        ("delete everything", lambda: delete(np.arange(len(mirror)))),
        ("grow from empty 1", lambda: append(1)),
        ("grow from empty 5000", lambda: append(5000)),
        ("grow from empty 7", lambda: append(7)),
    ]
    zero_fb = _check_state(mut, fresh, mirror, q, "initial")
    for what, step in steps:
        step()
        zero_fb += _check_state(mut, fresh, mirror, q, what)
    assert mut.fallback_count() - zero_fb == fb0, "a search other than the zero query went to the fallback"


def test_append_into_spare_capacity_refreshes_the_tensor_map(engines):
    mut, fresh = engines
    rng = np.random.default_rng(7)
    d = 256
    x = rng.standard_normal((9000, d)).astype(np.float32)
    mut.load_dense(x)
    mut.dense_reserve(20000)
    q = rng.standard_normal((16, d)).astype(np.float32)
    _search(mut, q, 10, 2)                       # caches the corpus map for n_pad = 9088
    new = rng.standard_normal((200, d)).astype(np.float32)
    new[100] = q[3]                             # row 9100: the unique best match of query 3, in the new tile 9088..9215
    rows = np.arange(9000, 9200)
    mut.dense_upsert(rows, new)
    best = 9100
    ids, sc, cnt = _search(mut, q, 10, 2)
    assert ids[3, 0] == best and sc[3, 0] > 0.999
    fresh.load_dense(np.concatenate([x, new]))
    for a, b in zip((ids, sc, cnt), _search(fresh, q, 10, 2)):
        assert np.array_equal(a, b)


def test_growth_with_and_without_reserve(built_lib):
    from sentio_b200.engine import B200Engine

    rng = np.random.default_rng(11)
    d = 1024
    chunks = [rng.standard_normal((m, d)).astype(np.float16) for m in (3000, 1, 4000, 127, 5000, 129, 2000)]
    q = _queries(rng, d)
    a, b, f = B200Engine(0), B200Engine(0), B200Engine(0)
    try:
        for e in (a, b):
            e.load_dense(np.zeros((0, d), np.float16))
        b.dense_reserve(20000)
        n = 0
        for c in chunks:
            for e in (a, b):
                e.dense_upsert(np.arange(n, n + len(c)), c)
            n += len(c)
        allx = np.concatenate(chunks)
        f.load_dense(allx)
        assert np.array_equal(a.dense_fetch(np.arange(n)), allx.astype(np.float32))
        assert np.array_equal(b.dense_fetch(np.arange(n)), allx.astype(np.float32))
        for mode in (1, 2):
            for B in (5, 260):
                ra, rb, rf = (_search(e, q[:B], 100, mode) for e in (a, b, f))
                for x, y, z in zip(ra, rb, rf):
                    assert np.array_equal(x, y) and np.array_equal(x, z)
    finally:
        for e in (a, b, f):
            e.close()


def _csr(conds):
    off = np.zeros(len(conds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in conds])
    return (off, np.asarray([f for c in conds for f, _ in c], np.int32),
            np.asarray([v for c in conds for _, v in c], np.int32))


def test_filtered_search_after_mutations(engines):
    mut, fresh = engines
    rng = np.random.default_rng(13)
    d, n0 = 256, 12000
    mirror = rng.standard_normal((n0, d)).astype(np.float32)

    def mk_tags(n):   # field 0: ~30 % code 0; field 1: ~1 % code 1 (gather path); field 2: parity
        u = rng.random(n)
        return {0: np.where(u < 0.3, 0, 1).astype(np.int32), 1: np.where(u < 0.01, 1, 0).astype(np.int32),
                2: (np.arange(n) % 2).astype(np.int32)}

    tags = mk_tags(n0)
    mut.load_dense(mirror)
    for f, c in tags.items():
        mut.load_dense_tags(f, c)
    q = _queries(rng, d)
    per_q = [[(0, 0)], [(1, 1)], [(0, 0), (2, 1)], [], [(1, 1), (2, 0)]]
    conds = lambda B: _csr([per_q[b % len(per_q)] for b in range(B)])

    # appends with their codes
    m = 3000
    rows = np.arange(n0, n0 + m)
    vec = rng.standard_normal((m, d)).astype(np.float32)
    mut.dense_upsert(rows, vec)
    nt = mk_tags(m)
    for f in tags:
        mut.dense_tags_write(f, rows, nt[f])
        tags[f] = np.concatenate([tags[f], nt[f]])
    mirror = np.concatenate([mirror, vec])
    _check_state(mut, fresh, mirror, q, "append + tags", tags, conds)
    # overwrites without a rewrite read -1
    rows = rng.choice(len(mirror), 500, replace=False)
    vec = rng.standard_normal((500, d)).astype(np.float32)
    mut.dense_upsert(rows, vec)
    mirror[rows] = vec
    for f in tags:
        tags[f][rows] = -1
    _check_state(mut, fresh, mirror, q, "overwrite", tags, conds)
    # codes travel with their rows through deletes
    for pick in (lambda n: rng.choice(n - 3000, 700, replace=False),
                 lambda n: np.r_[rng.choice(n - 900, 300, replace=False), np.arange(n - 900, n)]):
        dele = pick(len(mirror))
        mf, mt = mut.dense_delete(dele)
        keep = len(mirror) - len(dele)
        mirror[mt] = mirror[mf]
        mirror = mirror[:keep]
        for f in tags:
            tags[f][mt] = tags[f][mf]
            tags[f] = tags[f][:keep]
        _check_state(mut, fresh, mirror, q, "delete", tags, conds)
    # filtered results also match the oracle over the matching rows
    stored = dense_oracle.stored_rows(mirror)
    ids, sc, cnt = _search(mut, q[:16], 100, 2, conds(16))
    for b in range(16):
        msk = np.ones(len(mirror), bool)
        for f, v in per_q[b % len(per_q)]:
            msk &= tags[f] == v
        idx = np.flatnonzero(msk)
        wi, ws = dense_oracle.dense_topk(stored[idx], q[b], 100)
        assert_topk_matches(ids[b], sc[b], cnt[b], idx[wi], ws, what=f"filtered oracle q {b}")


def _fc(key, value):
    return NS(key=key, match=NS(value=value))


def test_vector_store_reference_call_sequence(built_lib):
    from sentio_b200.vector_store import B200VectorStore

    rng = np.random.default_rng(17)
    d = 128
    s = B200VectorStore(0)
    model = {}   # id -> (vector, payload), in no particular order

    def check(what):
        assert s.get_collection("kb").points_count == len(model)
        ids = list(model)
        q = rng.standard_normal((6, d)).astype(np.float32)
        stored = dense_oracle.stored_rows(np.stack([model[i][0] for i in ids])) if ids else None
        for flt in (None, _fc("metadata.source", "s1")):
            sel = [j for j, i in enumerate(ids) if flt is None or model[i][1]["metadata"]["source"] == "s1"]
            batch = s.search_batch("kb", q, limit=10, query_filter=flt)
            for b in range(6):
                hits = s.search("kb", q[b], limit=10, query_filter=flt)
                assert [(h.id, h.score) for h in hits] == [(h.id, h.score) for h in batch[b]]
                if sel:
                    wi, ws = dense_oracle.dense_topk(stored[sel], q[b], 10)
                    assert [h.id for h in hits] == [ids[sel[j]] for j in wi], what
                    assert np.allclose([h.score for h in hits], ws, rtol=1e-9, atol=1e-12)
                    assert all(h.payload == model[h.id][1] for h in hits)
                else:
                    assert hits == []
        recs, _ = s.scroll("kb", limit=100000)
        assert {r.id: r.payload for r in recs} == {i: p for i, (_v, p) in model.items()}
        some = ids[:5] + ["missing"]
        got = s.retrieve("kb", some, with_vectors=True)
        assert [r.id for r in got] == ids[:5]
        for r in got:
            assert np.array_equal(np.float32(r.vector), dense_oracle.stored_rows(model[r.id][0][None])[0].astype(np.float32))

    # _bootstrap_collection
    if not s.collection_exists("kb"):
        s.create_collection(collection_name="kb", vectors_config=NS(size=d, distance=NS(name="COSINE")))
    check("empty")
    # add_embeddings with default ids "0", "1", ...
    v = rng.standard_normal((300, d)).astype(np.float32)
    pts = [NS(id=str(i), vector=v[i].tolist(), payload={"content": f"c{i}", "metadata": {"source": f"s{i % 3}"}})
           for i in range(300)]
    assert s.upsert(collection_name="kb", points=pts).status == "completed"
    model.update({p.id: (v[i], p.payload) for i, p in enumerate(pts)})
    check("ingest")
    # re-ingest overwrites "0".. in place (and adds a few)
    w = rng.standard_normal((350, d)).astype(np.float32)
    pts = [NS(id=str(i), vector=w[i].tolist(), payload={"content": f"r{i}", "metadata": {"source": f"s{i % 2}"}})
           for i in range(350)]
    s.upsert(collection_name="kb", points=pts)
    model.update({p.id: (w[i], p.payload) for i, p in enumerate(pts)})
    check("re-ingest")
    # delete / delete_documents
    gone = [str(i) for i in rng.choice(350, 120, replace=False)] + ["nope"]
    s.delete(collection_name="kb", points_selector=NS(points=gone))
    for i in gone:
        model.pop(i, None)
    check("delete")
    s.close()


def test_search_in_flight_on_a_side_stream_sees_the_pre_delete_rows(engines):
    import torch

    mut, _ = engines
    rng = np.random.default_rng(19)
    d, n = 1024, 20000
    x = rng.standard_normal((n, d)).astype(np.float32)
    mut.load_dense(x)
    q = rng.standard_normal((256, d)).astype(np.float32)
    want = _oracle_top(dense_oracle.stored_rows(x), q, 10)
    qt = torch.from_numpy(q).cuda()
    mut.dense_topk_dev(qt, 10)   # sizes the scratch buffers: no reallocation (cudaFree synchronises) while enqueuing below
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        # ~50 ms of device delay ahead of the search: the delete below is issued while the search is still queued, so
        # only the delete's device synchronisation keeps it from moving the rows the search is about to read
        torch.cuda._sleep(100_000_000)
        ids, sc, cnt = mut.dense_topk_dev(qt, 10)
    assert not side.query(), "the side stream finished before the delete was issued"
    mut.dense_delete(np.unique(np.r_[[w[0][0] for w in want], np.arange(n - 3000, n)]))
    side.synchronize()
    ids, sc, cnt = ids.cpu().numpy(), sc.cpu().numpy(), cnt.cpu().numpy()
    for b in range(256):
        assert_topk_matches(ids[b], sc[b], cnt[b], want[b][0], want[b][1], what=f"in-flight q {b}")
