"""The full-pass epilogue of the wgmma scan (dense_mma.cu) at its edges: the survivor test of every score against its
query's threshold, the dead rows of the last tile, the filter's match bits, the Euclid and uint8 keys, and the
overflow of a survivor list.  Every result is checked against the fp64 oracle and, where a CUDA-core scan exists,
for byte identity with it."""
import numpy as np
import pytest

from helpers import assert_topk_matches
from metric_oracle import assert_metric_topk, magnitude, metric_topk, stored_metric
from u8_oracle import clustered_corpus, u8_magnitude, u8_topk_many

pytestmark = pytest.mark.gpu

N_TAIL = 9000 + 37        # >= 64 tiles (the wgmma scan's minimum), last tile 37 rows live and 91 dead


def _cosine(x16, Q):
    """fp64 cosine of every (row, query): [n, B]."""
    x = x16.astype(np.float64)
    q = np.asarray(Q, np.float32).astype(np.float64)
    den = np.sqrt((x * x).sum(1))[:, None] * np.sqrt((q * q).sum(1))[None, :]
    s = np.zeros((len(x), len(q)))
    np.divide(x @ q.T, den, out=s, where=den > 0)
    return s


def _want(s, b, k, rows=None):
    idx = np.arange(s.shape[0]) if rows is None else np.asarray(rows, np.int64)
    o = np.lexsort((idx, -s[idx, b]))[:k]
    return idx[o], s[idx[o], b]


def _both_scans(engine, q, k, **kw):
    """(wgmma scan result, CUDA-core scan result)."""
    try:
        engine.dense_set_mode(2)
        mma = engine.dense_topk(q, k, **kw)
        engine.dense_set_mode(1)
        core = engine.dense_topk(q, k, **kw)
    finally:
        engine.dense_set_mode(0)
    return mma, core


def _assert_identical(a, b, what):
    for x, y, name in zip(a, b, ("ids", "scores", "counts")):
        assert np.array_equal(x, y), f"{what}: {name} differ between the wgmma and the CUDA-core scan"


def _tail_corpus(seed, n=N_TAIL, d=128):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x16 = x.astype(np.float16)
    x16[300:700] = x16[17]           # 401 copies of one row: equal keys straddle rank k and the threshold
    x16[n - 20:] = x16[17]           # ... some of them in the live part of the last tile
    return x16, rng


@pytest.mark.parametrize("B", [16, 32, 64, 128, 256, 257])
def test_epilogue_every_group_width(engine, B):
    """One group of 16 .. 256 queries, and two groups (257).  Query 0 sits on the duplicate block, so hundreds of
    equal keys lie at rank k; query 1 is all zero (eps = 0, threshold 0, every score +-0: each row's key equals the
    threshold, and -0 >= +0 must pass)."""
    x16, rng = _tail_corpus(B)
    q = rng.standard_normal((B, x16.shape[1])).astype(np.float32)
    q[0] = x16[17].astype(np.float32)
    q[1] = 0.0
    engine.load_dense(x16)
    k = 50
    mma, core = _both_scans(engine, q, k)
    _assert_identical(mma, core, f"B={B}")
    s = _cosine(x16, q)
    for b in range(B):
        wi, ws = _want(s, b, k)
        assert_topk_matches(mma[0][b], mma[1][b], mma[2][b], wi, ws, what=f"B={B} b={b}")
    assert list(mma[0][1]) == list(range(k)), "the zero query ranks every row equal: the first k rows"


@pytest.mark.parametrize("B", [16, 256])
def test_epilogue_without_threshold_never_emits_dead_rows(engine, B):
    """k = 1024 exceeds the sampled keys of a 71-tile corpus, so the threshold is -inf and every live row survives.
    Every cosine is negative (positive rows, negative queries), so a dead row of the last tile (key 0) would rank
    first if the epilogue let it through."""
    rng = np.random.default_rng(5 + B)
    n, d, k = N_TAIL, 64, 1024
    x = np.abs(rng.standard_normal((n, d))).astype(np.float32) + 0.01
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x16 = x.astype(np.float16)
    q = -np.abs(rng.standard_normal((B, d))).astype(np.float32) - 0.01
    engine.load_dense(x16)
    mma, core = _both_scans(engine, q, k)
    _assert_identical(mma, core, f"B={B}")
    assert int(mma[0].max()) < n
    s = _cosine(x16, q)
    assert s.max() < 0.0
    for b in range(0, B, 5):
        wi, ws = _want(s, b, k)
        assert_topk_matches(mma[0][b], mma[1][b], mma[2][b], wi, ws, what=f"B={B} b={b}")


@pytest.mark.parametrize("frac", [1.0, 0.01])
def test_epilogue_filtered(engine, frac):
    """FILTER: every row matches, or ~1 % of them (still more than the 2048 rows the gather path takes, so the scan
    runs).  A duplicate block half inside the match set puts equal keys on both sides of the mask."""
    rng = np.random.default_rng(11)
    n, d, B, k = 300_000 + 37, 64, 256, 100
    x = rng.standard_normal((n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x16 = x.astype(np.float16)
    x16[1000:1400] = x16[3]
    tag = (rng.random(n) >= frac).astype(np.int32)   # 0 = match
    tag[1000:1200] = 0
    tag[1200:1400] = 1
    q = rng.standard_normal((B, d)).astype(np.float32)
    q[0] = x16[3].astype(np.float32)
    q[1] = 0.0
    engine.load_dense(x16)
    engine.load_dense_tags(0, tag)
    off = np.arange(B + 1, dtype=np.int32)
    flt = (off, np.zeros(B, np.int32), np.zeros(B, np.int32))
    mma, core = _both_scans(engine, q, k, filters=flt)
    _assert_identical(mma, core, f"frac={frac}")
    rows = np.flatnonzero(tag == 0)
    assert frac == 1.0 or len(rows) > 2048
    checked = [0, 1] + list(range(2, B, 16))
    s = _cosine(x16[rows], q[checked])
    for j, b in enumerate(checked):
        i, v = _want(s, j, k)
        assert_topk_matches(mma[0][b], mma[1][b], mma[2][b], rows[i], v, what=f"frac={frac} b={b}")


@pytest.mark.parametrize("B", [16, 256])
def test_epilogue_euclid(engine, B):
    """Euclid keys r (acc s) - h: rows of different norms, a duplicate block, the zero query."""
    rng = np.random.default_rng(21 + B)
    n, d, k = N_TAIL, 128, 100
    x = rng.standard_normal((n, d)).astype(np.float32) * rng.uniform(0.5, 2.0, (n, 1)).astype(np.float32)
    x[500:800] = x[9]
    q = rng.standard_normal((B, d)).astype(np.float32)
    q[0] = x[9]
    q[1] = 0.0
    engine.load_dense(x, metric="euclid")
    mma, core = _both_scans(engine, q, k)
    _assert_identical(mma, core, f"B={B}")
    y, c = stored_metric(x)
    rows = np.arange(n)
    for b in range(0, B, 3):
        wi, ws = metric_topk(y, c, q[b], k, "euclid")
        assert_metric_topk(mma[0][b], mma[1][b], mma[2][b], wi, ws, f"B={B} b={b}",
                           mag=magnitude(c, q[b], rows, "euclid"))


@pytest.mark.parametrize("metric", ["cosine", "euclid"])
def test_epilogue_uint8(engine, metric):
    """uint8 slots take the wgmma scan at every batch size; a clustered corpus puts many keys near the threshold."""
    n, d, B, k = N_TAIL, 128, 64, 100
    x = clustered_corpus(n, d, seed=31)
    x[200:600] = x[4]
    rng = np.random.default_rng(32)
    q = rng.standard_normal((B, d)).astype(np.float32)
    q[0] = x[4].astype(np.float32)
    engine.load_dense(x, metric=metric, storage="uint8")
    ids, sc, cnt = engine.dense_topk(q, k)
    want = u8_topk_many(x, q, k, metric)
    for b in range(B):
        assert_metric_topk(ids[b], sc[b], cnt[b], *want[b], f"{metric} b={b}", mag=u8_magnitude(x, q[b], metric))


def test_epilogue_overflowing_lists_take_the_fallback(engine):
    """Every row an exact copy of one: every key equals the k-th, all rows survive and each CTA's list overflows its
    capacity.  The queries must be flagged and answered by the brute-force kernel: the first k rows."""
    rng = np.random.default_rng(41)
    n, d, B, k = 300_000, 64, 32, 10
    row = rng.standard_normal(d).astype(np.float32)
    x16 = np.tile((row / np.linalg.norm(row)).astype(np.float16), (n, 1))
    q = rng.standard_normal((B, d)).astype(np.float32)
    engine.load_dense(x16)
    try:
        engine.dense_set_mode(2)
        fb0 = engine.fallback_count()
        ids, sc, cnt = engine.dense_topk(q, k)
        fb = engine.fallback_count() - fb0
    finally:
        engine.dense_set_mode(0)
    assert fb == B, f"{fb} of {B} queries took the fallback"
    s = _cosine(x16[:1], q)[0]
    for b in range(B):
        assert list(ids[b]) == list(range(k)) and int(cnt[b]) == k
        assert np.allclose(sc[b], s[b], rtol=1e-9, atol=1e-12)
