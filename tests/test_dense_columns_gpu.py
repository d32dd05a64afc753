"""Every per-row column of a dense slot through growth from an empty load, overwrites and deletes, for every storage and
metric: tag and value columns loaded on the still-empty slot (capacity 1), an upsert that grows the slot from capacity
0, an append that grows it again, overwrites that clear the payload, holes and tail deletes, deleting every row and
appending again.  After every step the mutated slot must equal, bit for bit, a slot freshly loaded with the same rows
and columns: stored rows, both scans, and a filtered search over a value range and two tag columns."""
import numpy as np
import pytest

from sentio_b200 import payload_filter as pf

pytestmark = pytest.mark.gpu

D = 256
TAGS = (0, 1)
VALS = (0, 1)


def _rows(rng, n, storage):
    if storage == "uint8":
        return rng.integers(0, 256, (n, D), dtype=np.uint8)
    x = rng.standard_normal((n, D)).astype(np.float32)
    return x * rng.uniform(0.5, 2.0, (n, 1)).astype(np.float32)


def _codes(rng, n):
    return rng.integers(-1, 6, n).astype(np.int32)


def _values(rng, n):
    v = rng.random(n)
    v[rng.random(n) < 0.2] = np.nan
    return v


def _pred(**kw):
    e = np.zeros(1, pf.PRED_DTYPE)
    for k, v in kw.items():
        e[0][k] = v
    return e


def _program(B):
    """value 0 in [0.2, 0.8] AND tag 0 == 2 AND tag 1 present, for every query"""
    one = np.concatenate([_pred(op=pf.RANGE, field=VALS[0], lo=0.2, hi=0.8, lo_incl=1, hi_incl=1),
                          _pred(op=pf.EQ, field=TAGS[0], a=2), _pred(op=pf.PRESENT, field=TAGS[1]),
                          _pred(op=pf.AND, a=3)])
    return (np.arange(B + 1, dtype=np.int32) * len(one), np.concatenate([one] * B), np.zeros(0, np.int32))


def _search(eng, q, k, mode):
    eng.dense_set_mode(mode)
    try:
        return eng.dense_topk(q, k)
    finally:
        eng.dense_set_mode(0)


def _check(mut, fresh, m, q, metric, storage, what):
    fresh.load_dense(m["x"], metric=metric, storage=storage)
    for f, c in m["tags"].items():
        fresh.load_dense_tags(f, c)
    for f, v in m["vals"].items():
        fresh.load_dense_values(f, v)
    n = len(m["x"])
    assert mut.dense_count[0] == n == fresh.dense_count[0], what
    if n:
        ids = np.arange(n)
        assert np.array_equal(mut.dense_fetch(ids), fresh.dense_fetch(ids)), f"{what}: stored rows"
    results = []
    for B, k in ((3, 10), (20, 50)):
        for mode in (1, 2):
            results.append((f"mode {mode} B {B} k {k}", _search(mut, q[:B], k, mode), _search(fresh, q[:B], k, mode)))
        if not m["vals"]:
            continue
        prog = _program(B)
        results.append((f"where B {B} k {k}", mut.dense_topk_where(q[:B], k, prog),
                        fresh.dense_topk_where(q[:B], k, prog)))
    for label, a, b in results:
        for u, v in zip(a, b):
            assert np.array_equal(u, v), f"{what}: {label} differs from a fresh load"
        if n == 0:
            assert np.all(a[2] == 0) and np.all(a[0] == -1), f"{what}: {label} on an empty slot"


def _write_payload(mut, m, rng, rows):
    for f in m["tags"]:
        c = _codes(rng, len(rows))
        mut.dense_tags_write(f, rows, c)
        m["tags"][f][rows] = c
    for f in m["vals"]:
        v = _values(rng, len(rows))
        mut.dense_values_write(f, rows, v)
        m["vals"][f][rows] = v


def _append(mut, m, rng, n, storage):
    x = _rows(rng, n, storage)
    n0 = len(m["x"])
    mut.dense_upsert(np.arange(n0, n0 + n), x)
    m["x"] = np.concatenate([m["x"], x])
    for f in m["tags"]:
        m["tags"][f] = np.concatenate([m["tags"][f], np.full(n, -1, np.int32)])
    for f in m["vals"]:
        m["vals"][f] = np.concatenate([m["vals"][f], np.full(n, np.nan)])
    return np.arange(n0, n0 + n)


def _delete(mut, m, rows):
    """delete `rows` and apply the returned plan to the mirrors"""
    mf, mt = mut.dense_delete(rows)
    keep = len(m["x"]) - len(rows)
    m["x"][mt] = m["x"][mf]
    m["x"] = m["x"][:keep]
    for col in (m["tags"], m["vals"]):
        for f in col:
            col[f][mt] = col[f][mf]
            col[f] = col[f][:keep]


@pytest.mark.parametrize("metric", ("cosine", "dot", "euclid"))
@pytest.mark.parametrize("storage", ("float16", "float32", "uint8"))
def test_columns_through_growth_and_deletes_equal_a_fresh_load(built_lib, storage, metric):
    from sentio_b200.engine import B200Engine

    rng = np.random.default_rng(7)
    q = rng.standard_normal((20, D)).astype(np.float32)
    dt = np.uint8 if storage == "uint8" else np.float32
    m = {"x": np.zeros((0, D), dt), "tags": {}, "vals": {}}   # mirrors of the rows and the loaded payload columns
    mut, fresh = B200Engine(0), B200Engine(0)
    try:
        mut.load_dense(m["x"], metric=metric, storage=storage)                       # 1. empty slot
        _check(mut, fresh, m, q, metric, storage, "empty load")
        for f in TAGS:                                                                # 2. payload at capacity 1
            m["tags"][f] = np.zeros(0, np.int32)
            mut.load_dense_tags(f, m["tags"][f])
        for f in VALS:
            m["vals"][f] = np.zeros(0)
            mut.load_dense_values(f, m["vals"][f])
        _check(mut, fresh, m, q, metric, storage, "payload on the empty slot")
        rows = _append(mut, m, rng, 9000, storage)                                    # 3. growth from capacity 0
        _write_payload(mut, m, rng, rows)
        _check(mut, fresh, m, q, metric, storage, "first growth")
        rows = _append(mut, m, rng, 4000, storage)                                    # 4. second growth
        _write_payload(mut, m, rng, rows[: len(rows) // 2])
        _check(mut, fresh, m, q, metric, storage, "second growth")
        over = rng.choice(len(m["x"]), 300, replace=False)                            # 5. overwrites clear payload
        x = _rows(rng, 300, storage)
        mut.dense_upsert(over, x)
        m["x"][over] = x
        for f in TAGS:
            m["tags"][f][over] = -1
        for f in VALS:
            m["vals"][f][over] = np.nan
        _check(mut, fresh, m, q, metric, storage, "overwrites")
        n = len(m["x"])                                                               # 6. holes + part of the tail
        dead = np.concatenate([rng.choice(n - 1000, 700, replace=False),
                               n - 1000 + rng.choice(1000, 400, replace=False)])
        _delete(mut, m, dead)
        _check(mut, fresh, m, q, metric, storage, "holes and tail")
        _delete(mut, m, np.arange(len(m["x"])))                                       # 7. every row
        _check(mut, fresh, m, q, metric, storage, "every row deleted")
        rows = _append(mut, m, rng, 500, storage)                                     # 8. append after emptying
        _write_payload(mut, m, rng, rows)
        _check(mut, fresh, m, q, metric, storage, "append after emptying")
    finally:
        mut.close()
        fresh.close()
