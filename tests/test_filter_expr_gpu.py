"""Boolean payload filters on the GPU (sb_dense_topk_where): the exact top-k of the matching rows for every metric and
storage, on the gather path, the masked scans, zero and all rows; a two-chunk batch of distinct programs; byte
identity with sb_dense_topk_filtered; value columns through upsert / delete / reserve; refused programs; and the store's
query_points end to end."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from f32_oracle import f32_magnitude, f32_max_norm, f32_topk
from filter_expr_oracle import matches
from metric_oracle import assert_metric_topk, magnitude, metric_topk, stored_metric
from sentio_b200 import payload_filter as pf

pytestmark = pytest.mark.gpu

N, D, K = 20000, 128, 20


def _payloads(rng, n):
    out = []
    for i in range(n):
        p = {"cat": f"c{rng.integers(40)}", "year": int(1990 + rng.integers(35)), "score": float(rng.random())}
        if i % 7 == 0:
            p["rare"] = "yes" if i % 49 == 0 else "no"      # 'yes' on ~400 rows: the gather path
        if i % 5 == 0:
            p["score"] = None
        if i % 11 == 0:
            p["year"] = True                                 # a bool is never numeric
        p["uid"] = i
        out.append(p)
    return out


def _fc(key, **m):
    return NS(key=key, match=NS(**m), range=None)


def _rg(key, **b):
    r = NS(gt=None, gte=None, lt=None, lte=None)
    for k, v in b.items():
        setattr(r, k, v)
    return NS(key=key, range=r, match=None)


FILTERS = [
    None,                                                                           # all rows (unfiltered)
    NS(must=[_rg("year", gte=1990)]),                                               # nearly all rows
    NS(should=[_fc("cat", value="c1"), _fc("cat", value="c2"), _fc("cat", value="c3")]),
    NS(must=[_fc("cat", any=[f"c{i}" for i in range(10)])], must_not=[_rg("score", lt=0.5)]),
    NS(must=[_fc("rare", value="yes")]),                                            # ~400 rows: gather
    NS(must=[_rg("score", gt=0.25, lte=0.2505)]),                                   # a few rows: gather
    NS(must=[_fc("cat", value="nope")]),                                            # zero rows
    NS(min_should=NS(conditions=[_fc("cat", value="c5"), _rg("year", lt=2000), _fc("rare", value="no")], min_count=2)),
    NS(must=[NS(should=[_rg("year", gte=2020), NS(must_not=[_fc("rare", value="no")])])]),
]


def _x(rng, n):
    x = rng.standard_normal((n, D)).astype(np.float32)
    return x * rng.uniform(0.5, 2.0, (n, 1)).astype(np.float32)


def _index(eng, payloads):
    return pf.PayloadIndex(payloads, lambda f, c: eng.load_dense_tags(f, c), lambda f, r, c: eng.dense_tags_write(f, r, c),
                           lambda f, v: eng.load_dense_values(f, v), lambda f, r, v: eng.dense_values_write(f, r, v))


def _oracle(x, q, rows, metric, storage):
    """(rows, scores, magnitude) of the exact fp64 top-K over `rows`: float32 storage scores x as given; float16
    storage scores the stored rows (Cosine: y = fp16(x / ||x||); Dot / Euclid: c * y)."""
    if storage == "float32":
        wi, ws = f32_topk(x, q, K, metric, rows=rows)
        return wi, ws, f32_magnitude(f32_max_norm(x), q, metric)
    y, c = stored_metric(x)
    if metric != "cosine":
        wi, ws = metric_topk(y, c, q, K, metric, rows=rows)
        return wi, ws, magnitude(c, q, wi, metric)
    y64, q64 = y[rows].astype(np.float64), np.asarray(q, np.float64)
    s = (y64 @ q64) / (np.sqrt((y64 * y64).sum(1)) * np.sqrt(q64 @ q64))
    o = np.lexsort((rows, -s))[:K]
    return rows[o], s[o], None


def _legacy_on_mask(eng, q, mask, field=15):
    """The exact top-k of the rows in `mask` through sb_dense_topk_filtered (a materialised tag column)."""
    eng.load_dense_tags(field, np.where(mask, 0, -1).astype(np.int32))
    one = np.ones(1, np.int32)
    return eng.dense_topk(q, K, filters=(np.array([0, 1], np.int32), one * field, one * 0))


@pytest.mark.parametrize("metric", ["cosine", "dot", "euclid"])
@pytest.mark.parametrize("storage", ["float16", "float32"])
def test_where_is_the_exact_topk_of_the_matching_rows(metric, storage):
    from sentio_b200.engine import B200Engine

    rng = np.random.default_rng(5)
    x, payloads = _x(rng, N), _payloads(rng, N)
    q = _x(rng, len(FILTERS))
    q[0] = 0.0                                                 # an all-zero query
    eng = B200Engine(0)
    try:
        eng.load_dense(x, metric=metric, storage=storage)
        progs = _index(eng, payloads).compile_programs(FILTERS)
        fb0 = eng.fallback_count()
        ids, sc, cnt = eng.dense_topk_where(q, K, progs)
        assert eng.fallback_count() == fb0
        for b, flt in enumerate(FILTERS):
            mask = np.array([matches(flt, p) for p in payloads])
            wi, ws, wc = _legacy_on_mask(eng, q[b], mask)
            assert int(cnt[b]) == int(wc[0]) == min(K, int(mask.sum())), b
            assert np.array_equal(ids[b], wi[0]) and np.array_equal(sc[b], ws[0]), b
            if b > 0:   # and the fp64 oracle over the stored representation (query 0 is the all-zero query)
                wi, ws, mag = _oracle(x, q[b], np.flatnonzero(mask), metric, storage)
                assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"{metric} {storage} q {b}", mag=mag)
    finally:
        eng.close()


def test_two_chunks_of_distinct_programs_and_empty_ones():
    from sentio_b200.engine import B200Engine

    rng = np.random.default_rng(9)
    x, payloads = _x(rng, N), _payloads(rng, N)
    filters = []
    for b in range(300):
        if b % 17 == 0:
            filters.append(None)
        else:
            lo = 1990 + b % 30
            filters.append(NS(must=[_rg("year", gte=lo, lt=lo + 1 + b % 4)], should=[_fc("cat", any=[f"c{b % 40}",
                                                                                                  f"c{(b * 7) % 40}"])]))
    q = _x(rng, 300)
    eng = B200Engine(0)
    try:
        eng.load_dense(x)
        fb0 = eng.fallback_count()
        ids, sc, cnt = eng.dense_topk_where(q, K, _index(eng, payloads).compile_programs(filters))
        for b in range(0, 300, 7):
            mask = np.array([matches(filters[b], p) for p in payloads])
            wi, ws, wc = _legacy_on_mask(eng, q[b], mask)
            assert cnt[b] == wc[0] and np.array_equal(ids[b], wi[0]) and np.array_equal(sc[b], ws[0]), b
        assert eng.fallback_count() == fb0
    finally:
        eng.close()


@pytest.mark.parametrize("shape", ["many_launches", "pool_in_global_memory"])
def test_chunks_beyond_the_shared_memory_budgets(shape):
    """A chunk whose distinct programs exceed the 1536 steps one launch stages (several launches, each writing only its
    own query columns; 200 queries leave padding columns too), and pools beyond the 8192 codes a launch stages (read
    from global memory)."""
    from sentio_b200.engine import B200Engine

    rng = np.random.default_rng(12)
    x, payloads = _x(rng, N), _payloads(rng, N)
    if shape == "many_launches":
        filters = [NS(should=[_fc("cat", value=f"c{b % 40}"), _fc("cat", value=f"c{(b * 3 + 1) % 40}"),
                              _rg("year", gte=1990 + b % 35, lte=1990 + (b * 7) % 35)],
                      must_not=[_rg("score", gt=(b % 10) / 10.0, lt=(b % 10) / 10.0 + 0.05)],
                      min_should=NS(conditions=[_fc("rare", value="no"), _rg("score", gte=0.5)], min_count=b % 2))
                   for b in range(200)]
    else:
        filters = [NS(must=[_fc("uid", any=[int(v) for v in rng.choice(N, 1000, replace=False)])],
                      should=[_fc("uid", any=[int(v) for v in rng.choice(N, 1000, replace=False)]),
                              _rg("score", lt=0.3)]) for _ in range(6)]
    q = _x(rng, len(filters))
    eng = B200Engine(0)
    try:
        eng.load_dense(x)
        off, prog, pool = _index(eng, payloads).compile_programs(filters)
        if shape == "many_launches":
            assert len(prog) > 1536 and len({bytes(prog[off[b]:off[b + 1]]) for b in range(len(filters))}) == 200
        else:
            assert len(pool) > 8192
        fb0 = eng.fallback_count()
        ids, sc, cnt = eng.dense_topk_where(q, K, (off, prog, pool))
        assert eng.fallback_count() == fb0
        for b, flt in enumerate(filters):
            rows = np.flatnonzero([matches(flt, p) for p in payloads])
            assert cnt[b] == min(K, len(rows)), b
            if b % 9 == 0 or shape != "many_launches":
                wi, ws, mag = _oracle(x, q[b], rows, "cosine", "float16")
                assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, f"{shape} q {b}", mag=mag)
    finally:
        eng.close()


def test_legacy_conjunctions_as_programs_are_byte_identical():
    from sentio_b200.engine import B200Engine

    rng = np.random.default_rng(2)
    x, payloads = _x(rng, N), _payloads(rng, N)
    filters = [NS(must=[_fc("cat", value=f"c{b % 40}")] + ([_fc("rare", value="no")] if b % 3 else []))
               for b in range(40)] + [NS(must=[_fc("cat", value="missing")]), None]
    q = _x(rng, len(filters))
    eng = B200Engine(0)
    try:
        eng.load_dense(x)
        idx = _index(eng, payloads)
        a = eng.dense_topk_where(q, K, idx.compile_programs(filters))
        f_off, fld, code = idx.compile(filters)
        b = eng.dense_topk(q, K, filters=(f_off, fld, code))
        for u, v in zip(a, b):
            assert np.array_equal(u, v)
    finally:
        eng.close()


def test_mutated_slot_equals_a_fresh_slot():
    from sentio_b200.engine import B200Engine

    rng = np.random.default_rng(4)
    x, payloads = _x(rng, 5000), _payloads(rng, 5000)
    filters = [NS(must=[_rg("score", gte=0.3)]), NS(must=[_rg("year", lt=2001)], must_not=[_fc("cat", value="c3")]),
               NS(must=[_fc("rare", value="yes")])]
    q = _x(rng, len(filters))
    a, b = B200Engine(0), B200Engine(0)
    try:
        a.load_dense(x)
        live = list(payloads)
        ia = _index(a, live)
        ia.compile_programs(filters)                        # indexes cat, rare, score, year
        a.dense_reserve(9000)
        new_x, new_p = _x(rng, 600), _payloads(rng, 600)
        rows = np.concatenate([np.arange(0, 600, 2), 5000 + np.arange(300)])
        enc = ia.encode(new_p)
        a.dense_upsert(rows, new_x)
        xs = np.concatenate([x, np.zeros((300, D), np.float32)])
        live.extend([None] * 300)
        for r, p, v in zip(rows.tolist(), new_p, new_x):
            live[r] = p
            xs[r] = v
        ia.apply(rows, enc)
        dead = rng.choice(len(live), 700, replace=False)
        mf, mt = a.dense_delete(dead)
        for f_, t_ in zip(mf.tolist(), mt.tolist()):
            live[t_] = live[f_]
            xs[t_] = xs[f_]
        keep = len(live) - len(dead)
        del live[keep:]
        xs = xs[:keep]
        b.load_dense(xs)
        ib = _index(b, live)
        got = a.dense_topk_where(q, K, ia.compile_programs(filters))
        want = b.dense_topk_where(q, K, ib.compile_programs(filters))
        for u, v in zip(got, want):
            assert np.array_equal(u, v)
    finally:
        a.close()
        b.close()


def _pred(**kw):
    e = np.zeros(1, pf.PRED_DTYPE)
    for k, v in kw.items():
        e[0][k] = v
    return e


@pytest.mark.parametrize("prog, pool", [
    (_pred(op=99), []),
    (_pred(op=pf.EQ, field=9, a=0), []),                                    # tag field not loaded
    (_pred(op=pf.RANGE, field=3, lo=0.0, hi=1.0), []),                      # value field not loaded
    (_pred(op=pf.EQ, field=0, a=-1), []),
    (_pred(op=pf.IN, field=0, a=0, b=3), [1, 2]),                           # pool range out of bounds
    (_pred(op=pf.IN, field=0, a=0, b=2), [2, 1]),                           # not ascending
    (_pred(op=pf.RANGE, field=0, lo=np.nan, hi=1.0, lo_incl=1, hi_incl=1), []),
    (np.concatenate([_pred(op=pf.EQ, field=0, a=0), _pred(op=pf.EQ, field=0, a=1)]), []),   # two entries left
    (_pred(op=pf.AND, a=1), []),                                            # pops an empty stack
    (np.concatenate([_pred(op=pf.PRESENT, field=0)] * 65 + [_pred(op=pf.AND, a=65)]), []),  # stack > 64
    (np.concatenate([_pred(op=pf.PRESENT, field=0)] + [_pred(op=pf.AND, a=1)] * 1024), []),  # > 1024 steps
])
def test_malformed_programs_are_refused_and_change_nothing(prog, pool):
    from sentio_b200._lib import SentioB200Error
    from sentio_b200.engine import B200Engine

    rng = np.random.default_rng(1)
    x = _x(rng, 3000)
    eng = B200Engine(0)
    try:
        eng.load_dense(x)
        eng.load_dense_tags(0, (np.arange(3000) % 4).astype(np.int32))
        eng.load_dense_values(0, rng.random(3000))
        q = _x(rng, 2)
        good = (np.array([0, 1, 1], np.int32), _pred(op=pf.EQ, field=0, a=2), np.zeros(0, np.int32))
        before = eng.dense_topk_where(q, K, good)
        progs = (np.array([0, 1, 1 + len(prog)], np.int32), np.concatenate([_pred(op=pf.EQ, field=0, a=2), prog]),
                 np.asarray(pool, np.int32))
        with pytest.raises(SentioB200Error):
            eng.dense_topk_where(q, K, progs)
        after = eng.dense_topk_where(q, K, good)
        for u, v in zip(before, after):
            assert np.array_equal(u, v)
    finally:
        eng.close()


def test_store_query_points_end_to_end():
    from sentio_b200.vector_store import B200VectorStore, VectorParams

    rng = np.random.default_rng(8)
    x, payloads = _x(rng, 3000), _payloads(rng, 3000)
    s = B200VectorStore(0)
    try:
        s.create_collection("c", x, ids=[f"p{i}" for i in range(3000)], payloads=payloads,
                            vectors_config=VectorParams(D, "Dot"))
        flt = FILTERS[3]
        res = s.query_points("c", x[10], query_filter=flt, limit=15, offset=5).points
        rows = [i for i, p in enumerate(payloads) if matches(flt, p)]
        sc = x[rows].astype(np.float64) @ x[10].astype(np.float64)
        want = [f"p{rows[i]}" for i in np.argsort(-sc, kind="stable")[5:20]]
        assert [p.id for p in res] == want
        batch = s.query_batch_points("c", [NS(query=x[10], filter=flt, limit=15, offset=5, score_threshold=None,
                                              with_payload=False), NS(query=x[11], filter=None, limit=3, offset=None,
                                                                      score_threshold=None, with_payload=True)])
        assert [p.id for p in batch[0].points] == want and batch[0].points[0].payload is None
        assert [p.id for p in batch[1].points] == [p.id for p in s.query_points("c", x[11], limit=3).points]
    finally:
        s.close()
