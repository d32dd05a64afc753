"""wgmma scan with groups of 256 queries: several full groups in one batch, and the widest row length."""
import numpy as np
import pytest

from helpers import assert_topk_matches
from oracle import dense as dense_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,d,k,B", [(30000, 1024, 100, 512), (10000, 4096, 50, 256)])
def test_dense_full_query_groups_match_oracle_and_cuda_core_scan(engine, n, d, k, B):
    """B = 512 is two 256-query groups; d = 4096 with B = 256 streams 64 query boxes per tile.  Results must equal the
    oracle AND be bit-identical to the CUDA-core scan."""
    rng = np.random.default_rng(n + d + B)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x16 = x.astype(np.float16)
    x16[100:140] = x16[50]                  # a block of exact duplicates
    q = rng.standard_normal((B, d)).astype(np.float32)
    q[3] = x16[50].astype(np.float32)       # exact ties
    q[5] = 0.0                              # zero query
    q[B - 1] = x16[n - 1].astype(np.float32)   # last row of the corpus, last query of the last group
    engine.load_dense(x16, id_base=7)
    engine.dense_set_mode(0)
    ids, sc, cnt = engine.dense_topk(q, k)
    for b, (wi, ws) in enumerate(dense_oracle.dense_topk_multi(x16, q, k)):
        assert_topk_matches(ids[b] - 7, sc[b], cnt[b], wi, ws, what=f"n={n} d={d} k={k} b={b}")
    engine.dense_set_mode(1)
    try:
        ids1, sc1, cnt1 = engine.dense_topk(q, k)
    finally:
        engine.dense_set_mode(0)
    assert np.array_equal(ids, ids1) and np.array_equal(sc, sc1) and np.array_equal(cnt, cnt1)
    assert ids[B - 1, 0] - 7 == n - 1
