"""Recommendation by example on the device (DESIGN.md K1j) against the fp64 oracle on the stored rows
(tests/reco_oracle.py): every storage x {Cosine, Dot} x {best_score, sum_scores}, ragged and 1024 dimensions, positives
only / negatives only / both, batches spanning several passes, filter programs, mutated slots, exact duplicates that
must take the brute force, sum_scores of one positive equal to query_points, and average_vector on every distance."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from metric_oracle import assert_metric_topk
from reco_oracle import reco_topk, stored, similarities

pytestmark = pytest.mark.gpu


def corpus(n, d, storage, seed):
    rng = np.random.default_rng(seed)
    if storage == "uint8":
        return rng.integers(0, 256, (n, d)).astype(np.uint8)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x *= rng.uniform(0.5, 2.0, (n, 1)).astype(np.float32)
    return x


def examples(x, rng, m):
    d = x.shape[1]
    ex = rng.standard_normal((m, d)).astype(np.float32)
    if x.dtype == np.uint8:
        ex = ex * 40 + 128
    take = rng.integers(0, len(x), m)
    near = rng.random(m) < 0.5
    ex[near] = x[take[near]].astype(np.float32) + ex[near] * 0.05   # examples close to stored rows
    return ex.astype(np.float32)


def check(engine, x, storage, metric, ex, r_off, n_pos, strategies, k, what, cand=None, programs=None):
    ids, sc, cnt = engine.dense_recommend(ex, r_off, n_pos, strategies, k, programs=programs)
    rows, fac = stored(x, storage, metric)
    for r in range(len(n_pos)):
        e = ex[r_off[r]:r_off[r + 1]]
        wi, ws = reco_topk(rows, fac, e, n_pos[r], strategies[r], metric, k, None if cand is None else cand[r])
        mag = sum(float(np.abs(similarities(rows, fac, v, metric)).max()) for v in e)
        assert_metric_topk(ids[r], sc[r], cnt[r], wi, ws, f"{what} request {r}", mag=mag)


@pytest.mark.parametrize("storage", ["float16", "float32", "uint8"])
@pytest.mark.parametrize("metric", ["cosine", "dot"])
@pytest.mark.parametrize("d", [200, 1024])
def test_storage_metric_strategy(engine, storage, metric, d):
    x = corpus(9000, d, storage, seed=d)
    engine.load_dense(x, metric=metric, storage=storage)
    rng = np.random.default_rng(7)
    sizes = [(3, 0), (0, 2), (4, 3), (1, 1), (8, 0)]
    ex = examples(x, rng, sum(p + q for p, q in sizes))
    r_off = np.cumsum([0] + [p + q for p, q in sizes])
    n_pos = [p for p, _ in sizes]
    fb0 = engine.fallback_count()
    for strategy in ("best_score", "sum_scores"):
        check(engine, x, storage, metric, ex, r_off, n_pos, [strategy] * len(sizes), 100, f"{storage} {metric} {d}")
    assert engine.fallback_count() == fb0


@pytest.mark.parametrize("total", [1, 255, 256, 257, 600])
def test_batches_across_passes(engine, total):
    x = corpus(5000, 64, "float16", seed=3)
    engine.load_dense(x)
    rng = np.random.default_rng(total)
    sizes = []
    left = total
    while left:
        m = int(min(left, rng.integers(1, 40) if total > 1 else 1))
        sizes.append(m)
        left -= m
    ex = examples(x, rng, total)
    r_off = np.cumsum([0] + sizes)
    n_pos = [int(rng.integers(0, m + 1)) for m in sizes]
    strategies = ["best_score" if i % 2 else "sum_scores" for i in range(len(sizes))]
    check(engine, x, "float16", "cosine", ex, r_off, n_pos, strategies, 10, f"total {total}")


def test_filter_programs(engine):
    from sentio_b200.payload_filter import PayloadIndex

    x = corpus(9000, 128, "float32", seed=5)
    engine.load_dense(x, metric="dot", storage="float32")
    payloads = [{"year": 2000 + i % 30, "src": f"s{i % 7}"} for i in range(len(x))]
    pi = PayloadIndex(payloads, lambda f, c: engine.load_dense_tags(f, c), None,
                      lambda f, v: engine.load_dense_values(f, v), None)
    flts = [NS(must=[NS(key="year", range=NS(gt=None, gte=2025, lt=None, lte=None), match=None)]),
            None,
            NS(should=[NS(key="src", match=NS(any=["s1", "s3"]))], must_not=[NS(key="year", match=NS(value=2001))])]
    from filter_expr_oracle import matches
    cand = [np.array([i for i in range(len(x)) if f is None or matches(f, payloads[i])]) for f in flts]
    rng = np.random.default_rng(2)
    ex = examples(x, rng, 9)
    check(engine, x, "float32", "dot", ex, [0, 3, 6, 9], [2, 1, 0], ["best_score", "sum_scores", "best_score"], 50,
          "filtered", cand=cand, programs=pi.compile_programs(flts))


def test_duplicates_take_the_brute_force(engine):
    x = corpus(9000, 64, "float16", seed=9)
    x[:3000] = x[0]
    engine.load_dense(x)
    fb0 = engine.fallback_count()
    ex = np.stack([x[0] + 0.01, x[5000]]).astype(np.float32)
    check(engine, x, "float16", "cosine", ex, [0, 2], [1], ["sum_scores"], 100, "duplicates")
    assert engine.fallback_count() > fb0


@pytest.fixture
def store(built_lib):
    from sentio_b200.vector_store import B200VectorStore

    s = B200VectorStore(0)
    yield s
    s.close()


@pytest.mark.parametrize("dist", ["Cosine", "Dot"])
def test_one_positive_sum_scores_is_query_points(store, dist):
    from sentio_b200.vector_store import VectorParams

    x = corpus(9000, 96, "float16", seed=11)
    store.create_collection("c", x, vectors_config=VectorParams(96, dist))
    q = np.random.default_rng(1).standard_normal(96).astype(np.float32)
    got = store.recommend("c", positive=[q], strategy="sum_scores", limit=50)
    want = store.query_points("c", q, limit=50).points
    assert [(p.id, p.score) for p in got] == [(p.id, p.score) for p in want]


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid"])
def test_average_vector_is_a_nearest_query(store, dist):
    from sentio_b200.vector_store import VectorParams

    x = corpus(9000, 64, "float16", seed=12)
    store.create_collection("c", x, vectors_config=VectorParams(64, dist))
    got = store.recommend("c", positive=["3", "8"], negative=["20"], limit=30)
    v = np.asarray([r.vector for r in store.retrieve("c", ["3", "8", "20"], with_vectors=True)], np.float64)
    ap = (v[0] + v[1]) / 2
    q = (ap + (ap - v[2])).astype(np.float32)
    want = [p for p in store.query_points("c", q, limit=33).points if p.id not in ("3", "8", "20")][:30]
    assert [(p.id, p.score) for p in got] == [(p.id, p.score) for p in want]


def test_after_upsert_and_delete(store):
    from sentio_b200.vector_store import VectorParams

    x = corpus(9000, 64, "uint8", seed=13)
    store.create_collection("c", x, vectors_config=VectorParams(64, "Dot", "uint8"))
    rng = np.random.default_rng(4)
    store.upsert("c", [NS(id=str(i), vector=rng.integers(0, 256, 64).astype(np.float32), payload={})
                       for i in range(0, 9000, 97)])
    store.delete("c", [str(i) for i in range(1, 9000, 89)])
    ids = [r.id for r in store.scroll("c", limit=20000)[0]]
    rows = np.asarray([r.vector for r in store.retrieve("c", ids, with_vectors=True)], np.float64)
    ex = examples(x, rng, 4)
    got = store.recommend("c", positive=[ex[0], ex[1], "5"], negative=[ex[2]], strategy="best_score", limit=40)
    e5 = rows[ids.index("5")].astype(np.float32)
    wi, ws = reco_topk(rows, None, [ex[0], ex[1], e5, ex[2]], 3, "best_score", "dot", 41)
    want = [(ids[i], s) for i, s in zip(wi, ws) if ids[i] != "5"][:40]
    assert [p.id for p in got] == [w[0] for w in want]
    assert np.allclose([p.score for p in got], [w[1] for w in want], rtol=1e-12)


def branch_band(storage, n=9000, d=256, band=600, seed=21):
    """(rows, positive example, negative example): e+- = m +- w with w orthogonal to m and ||e+|| = ||e-||, and `band`
    rows m + t w (+ the storage's rounding) that are the best rows of both examples, whose similarities to e+ and e-
    differ by far less than the scan's error bound (p - n = 2 t ||w||^2 for Dot), on both sides of p = n and at it."""
    rng = np.random.default_rng(seed)
    if storage == "uint8":
        m = np.full(d, 128.0)
        w = np.zeros(d)
        w[0], w[1] = 1e-3, -1e-3
        x = rng.integers(0, 256, (n, d))
        b = np.full((band, d), 200) + rng.integers(-2, 3, (band, d))
        b[:, 1] = b[:, 0] + rng.integers(-1, 2, band)   # x0 - x1 in {-1, 0, 1}: p - n in {-2, 0, 2} x 1e-3 x 128 / ...
        x[:band] = b
        x = x.astype(np.uint8)
    else:
        m = rng.standard_normal(d)
        w = rng.standard_normal(d)
        w -= (w @ m) / (m @ m) * m
        w *= 0.01 * np.linalg.norm(m) / np.linalg.norm(w)
        x = rng.standard_normal((n, d)) * 0.3 * np.linalg.norm(m) / np.sqrt(d)
        t = rng.uniform(-0.05, 0.05, band)[:, None]
        r = rng.standard_normal((band, d))
        r -= np.outer(r @ m / (m @ m), m) + np.outer(r @ w / (w @ w), w)   # spread the band's cosines, not p - n
        r *= (rng.uniform(0.0, 0.02, band) * np.linalg.norm(m) / np.linalg.norm(r, axis=1))[:, None]
        x[:band] = m[None, :] * rng.uniform(0.9, 1.1, band)[:, None] + t * w[None, :] + r
        x = x.astype(np.float32)
    return x, (m + w).astype(np.float32), (m - w).astype(np.float32)


@pytest.mark.parametrize("metric", ["cosine", "dot"])
@pytest.mark.parametrize("storage", ["float16", "uint8"])
def test_branch_window_adversarial(engine, metric, storage):
    """The k-th score lies among rows whose p - n is far inside the window: the approximate keys put many of them on the
    wrong side of best_score's jump at p = n.  A delta that is too small, or an interval that ignores the jump, loses
    rows of the exact top-k; sum_scores sees the same near-cancelling rows."""
    x, e_pos, e_neg = branch_band(storage)
    engine.load_dense(x, metric=metric, storage=storage)
    ex = np.stack([e_pos, e_neg])
    rows, fac = stored(x, storage, metric)
    s = np.stack([similarities(rows, fac, e, metric) for e in ex], 1)
    top = np.argsort(-s[:, 0], kind="stable")[:300]
    assert (top < 600).all()
    assert (s[top, 0] > s[top, 1]).sum() >= 100 and (s[top, 0] <= s[top, 1]).sum() >= 50
    for strategy in ("best_score", "sum_scores"):
        check(engine, x, storage, metric, ex, [0, 2], [1], [strategy], 100, f"band {storage} {metric} {strategy}")
