"""The adversarial window corpora of tests/window_oracle.py on the device: the exact top-k of every adversarial query
is a set of decoys whose scan error pushes them between a_k - 2 eps and a_k - eps, so a window or an eps narrower than
the one DESIGN.md K1 derives returns baits instead.  Ids and scores must equal the fp64 oracles, no query may take the
brute-force fallback (it would hide a wrong eps), and on float32 cases a float16 slot of the same rows must answer
differently (the float32 exactness is not vacuous).  The crowded case must take the fallback and stay exact."""
import numpy as np
import pytest

import window_oracle as wo
from f32_oracle import f32_magnitude, f32_max_norm, f32_topk_many
from helpers import assert_topk_matches
from metric_oracle import assert_metric_topk, magnitude, metric_topk, stored_metric
from oracle import dense as dense_oracle
from u8_oracle import u8_magnitude, u8_topk_many

pytestmark = pytest.mark.gpu

RUNS = {"mma": ((2, 16), (2, 256)), "core": ((1, 3),)}   # (dense_set_mode, B)


@pytest.fixture(scope="module")
def engines(built_lib):
    from sentio_b200.engine import B200Engine

    a, b = B200Engine(0), B200Engine(0)
    yield a, b
    a.close()
    b.close()


def _want(case, B):
    """Per query (ids, scores) of the fp64 oracle on the slot's scored representation, and the magnitude for
    assert_metric_topk."""
    q, k, rows = case.q[:B], case.k, None if case.match is None else np.flatnonzero(case.match)
    if case.storage == "float32":
        xmax = f32_max_norm(case.x)
        return [(w, f32_magnitude(xmax, q[b], case.metric)) for b, w in
                enumerate(f32_topk_many(case.x, q, k, case.metric, rows=rows))]
    if case.storage == "uint8":
        return [(w, u8_magnitude(case.x, q[b], case.metric)) for b, w in
                enumerate(u8_topk_many(case.x, q, k, case.metric, rows=rows))]
    if case.metric == "cosine":
        stored = dense_oracle.stored_rows(case.x)
        out = []
        for b in range(B):
            s = dense_oracle.cosine_scores(stored, q[b])
            idx = np.arange(len(s)) if rows is None else rows
            o = idx[np.lexsort((idx, -s[idx]))[:k]]
            out.append(((o, s[o]), None))
        return out
    y, c = stored_metric(case.x)
    allr = np.arange(len(y)) if rows is None else rows
    return [(metric_topk(y, c, q[b], k, case.metric, rows=rows), magnitude(c, q[b], allr, case.metric))
            for b in range(B)]


def _load(eng, case):
    if case.x0 is not None:
        eng.load_dense(case.x0, metric=case.metric, storage=case.storage)
        eng.dense_upsert(case.up_rows, case.x[case.up_rows])
    else:
        eng.load_dense(case.x, metric=case.metric, storage=case.storage)
    if case.match is not None:
        eng.load_dense_tags(0, case.match.astype(np.int32))


def _filters(case, B):
    if case.match is None:
        return None
    return (np.arange(B + 1, dtype=np.int32), np.zeros(B, np.int32), np.ones(B, np.int32))


def _search(eng, case, mode, B):
    eng.dense_set_mode(mode)
    try:
        return eng.dense_topk(case.q[:B], case.k, filters=_filters(case, B))
    finally:
        eng.dense_set_mode(0)


@pytest.mark.parametrize("name", sorted(wo.CASES))
def test_window_holds_the_exact_top_k(engines, name):
    eng, f16 = engines
    case = wo.adversarial_case(name)
    _load(eng, case)
    want = _want(case, wo.B_MAX)
    for scan in case.scans:
        for mode, B in RUNS[scan]:
            fb0 = eng.fallback_count()
            ids, sc, cnt = _search(eng, case, mode, B)
            assert eng.fallback_count() == fb0, f"{name} {scan} B {B}: a query took the brute-force fallback"
            for b in range(B):
                (wi, ws), mag = want[b]
                what = f"{name} {scan} B {B} q {b}"
                if mag is None:
                    assert_topk_matches(ids[b], sc[b], cnt[b], wi, ws, what=what)
                else:
                    assert_metric_topk(ids[b], sc[b], cnt[b], wi, ws, what, mag=mag)
            for m in range(wo.N_ADV):   # the adversarial answer is the decoys
                assert sorted(ids[m].tolist()) == sorted(case.bands[m][0].tolist()), f"{name} {scan} B {B} q {m}"
    if case.storage == "float32":
        f16.load_dense(case.x, metric=case.metric)
        if case.match is not None:
            f16.load_dense_tags(0, case.match.astype(np.int32))
        ids16, _, _ = _search(f16, case, 2, 16)
        ids32, _, _ = _search(eng, case, 2, 16)
        assert any(set(ids16[m].tolist()) != set(ids32[m].tolist()) for m in range(wo.N_ADV)), \
            f"{name}: the float16 slot of the same rows must answer differently"


@pytest.mark.parametrize("mode, B", [(1, 3), (2, 16)])
def test_crowded_window_takes_the_fallback_and_stays_exact(engines, mode, B):
    eng, _ = engines
    x, q, rows = wo.crowded_case()
    eng.load_dense(x)
    stored = dense_oracle.stored_rows(x)
    fb0 = eng.fallback_count()
    eng.dense_set_mode(mode)
    try:
        ids, sc, cnt = eng.dense_topk(q[:B], 10)
    finally:
        eng.dense_set_mode(0)
    assert eng.fallback_count() - fb0 >= wo.N_ADV, "a list full of window rows must send its query to the fallback"
    for b in range(B):
        wi, ws = dense_oracle.topk(dense_oracle.cosine_scores(stored, q[b]), 10)
        assert_topk_matches(ids[b], sc[b], cnt[b], wi, ws, what=f"crowded mode {mode} q {b}")
    for m in range(wo.N_ADV):
        assert ids[m].tolist() == sorted(rows.tolist())[:10], "exact duplicates: ties by ascending row"
