"""The filtered-BM25 reference of tests/bm25_filter_oracle.py against brute force on small inputs: ties, zero and
negative scores, empty and unknown-value conditions, k larger than the matches."""
import numpy as np
import pytest

import bm25_filter_oracle as fo


def _brute(scores, tags, conds, k):
    n = len(scores)
    keep = [i for i in range(n) if all(c >= 0 and tags[f][i] == c for f, c in conds) and scores[i] > 0]
    return sorted(keep, key=lambda i: (-scores[i], i))[:k]


@pytest.mark.parametrize("seed", range(20))
def test_filtered_topk_equals_brute_force(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 300))
    scores = rng.choice([-1.0, 0.0, 0.5, 1.25, 2.0, 3.5], n) + rng.choice([0.0, 0.0, 1e-3], n)   # many exact ties
    tags = {f: rng.integers(-1, 4, n).astype(np.int32) for f in range(3)}
    for conds in ([], [(0, 1)], [(0, 2), (1, 0)], [(0, 1), (1, 2), (2, 3)], [(1, -1)], [(2, 9)]):
        for k in (1, 5, 50, 400):
            m = fo.match_mask(tags, conds, n)
            assert fo.filtered_topk(scores, m, k).tolist() == _brute(scores, tags, conds, k), (seed, conds, k)


def test_csr_and_padding_layout():
    off, fld, code = fo.csr([[], [(0, 3), (2, -1)], [(1, 0)]])
    assert off.tolist() == [0, 0, 2, 3] and fld.tolist() == [0, 2, 1] and code.tolist() == [3, -1, 0]
    assert off.dtype == fld.dtype == code.dtype == np.int32
    s = np.array([0.0, 2.0, 1.0])
    ids, sc, cnt = fo.padded([np.array([1, 2]), np.array([], np.int64)], [s, s], 3, id_base=10)
    assert ids.tolist() == [[11, 12, -1], [-1, -1, -1]] and sc.tolist() == [[2.0, 1.0, 0.0], [0.0] * 3]
    assert cnt.tolist() == [2, 0]
