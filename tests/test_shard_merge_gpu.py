"""K6 parity: sb_merge_shards_dev over an all-gathered record buffer in the pipeline's own byte layout
(HybridPipeline._record_layout / _views, two signals per record, signal 1 at a nonzero base offset) == the merge
oracle (union of every shard's first `count` entries, score desc in K1's total order, id asc, cut to k), exactly."""
import numpy as np
import pytest

import small_kernels_oracle as so

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pipe(engine):
    from sentio_b200.pipeline import HybridPipeline

    return HybridPipeline(0, engine=engine)


def _records_buffer(pipe, cases, G, B, k):
    """cases[sig] = (ids [G,B,k], scores [G,B,k], counts [G,B]) -> one [G, record bytes] uint8 CUDA buffer."""
    import torch

    _, nbytes = pipe._record_layout(B, k, len(cases))
    buf = torch.zeros((G, nbytes), dtype=torch.uint8, device="cuda:0")
    for sig, (ids, sc, cnt) in enumerate(cases):
        for g in range(G):
            v_ids, v_sc, v_cnt = pipe._views(buf[g], B, k, sig)
            v_ids.copy_(torch.from_numpy(ids[g]))
            v_sc.copy_(torch.from_numpy(sc[g]))
            v_cnt.copy_(torch.from_numpy(cnt[g]))
    return buf, nbytes


def _merge(pipe, buf, nbytes, G, B, k, sig):
    import torch

    out = pipe.engine.merge_shards_dev(*pipe._views(buf[0], B, k, sig), nbytes, G)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


@pytest.mark.parametrize("G", [1, 2, 3, 8])
@pytest.mark.parametrize("k", [1, 100, 1024])
def test_merge_equals_oracle(pipe, G, k):
    B = 37 if k < 1024 else 11
    cases, want = [], []
    for sig in range(2):
        rec, exp = so.merge_case(1000 * G + k + sig, G, B, k)
        cases.append(rec)
        want.append(exp)
    buf, nbytes = _records_buffer(pipe, cases, G, B, k)
    for sig in range(2):
        ids, sc, cnt = _merge(pipe, buf, nbytes, G, B, k, sig)
        w_ids, w_sc, w_cnt = want[sig]
        assert np.array_equal(cnt, w_cnt), (G, k, sig)
        assert np.array_equal(ids, w_ids), (G, k, sig)
        # bit patterns: +0.0 and -0.0 are different scores here
        assert np.array_equal(sc.view(np.uint64), w_sc.view(np.uint64)), (G, k, sig)


def test_merge_ties_across_shards_at_rank_k(pipe):
    """Hand case: every shard holds the same score at its boundary; the lowest ids win across shards, +0.0 outranks
    -0.0 whatever the ids, and nothing past a count is read."""
    G, B, k = 3, 2, 4
    ids = np.asarray([[[30, 31, 32, 33], [5, 6, 7, 8]],
                      [[10, 11, 12, 13], [50, 51, 52, 53]],
                      [[20, 21, 22, 23], [1, 2, 3, 4]]], np.int64)
    sc = np.asarray([[[1.0, 0.5, 0.5, 0.5], [0.0, 0.0, -0.0, 9.0]],
                     [[0.5, 0.5, 9.0, 9.0], [0.0, -0.0, -0.0, -0.0]],
                     [[0.5, 0.5, 0.5, 0.5], [-0.0, -0.0, -0.0, -0.0]]])
    cnt = np.asarray([[4, 3], [2, 4], [4, 4]], np.int32)
    want = so.merge_oracle((ids, sc, cnt), G, k)
    assert want[0].tolist() == [[30, 10, 11, 20], [5, 6, 50, 1]]
    buf, nbytes = _records_buffer(pipe, [(ids, sc, cnt)], G, B, k)
    got = _merge(pipe, buf, nbytes, G, B, k, 0)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2])
    assert np.array_equal(got[1].view(np.uint64), want[1].view(np.uint64))


def test_merge_all_counts_zero_pads(pipe):
    G, B, k = 2, 5, 100
    rec, want = so.merge_case(9, G, B, k)
    rec = (rec[0], rec[1], np.zeros_like(rec[2]))
    buf, nbytes = _records_buffer(pipe, [rec], G, B, k)
    ids, sc, cnt = _merge(pipe, buf, nbytes, G, B, k, 0)
    assert (cnt == 0).all() and (ids == -1).all() and np.array_equal(sc.view(np.uint64), np.zeros((B, k), np.uint64))


def test_merge_beyond_shared_memory_is_unsupported(pipe):
    """G*k = 8200 rounds up to a 16384-entry sort (256 KB) > the opt-in shared memory: refused on the host, before any
    launch.  G*k = 8192 (the previous test's G = 8, k = 1024) is the largest accepted size."""
    from sentio_b200._lib import SentioB200Error

    G, B, k = 8, 1, 1025
    rec = (np.zeros((G, B, k), np.int64), np.zeros((G, B, k)), np.zeros((G, B), np.int32))
    buf, nbytes = _records_buffer(pipe, [rec], G, B, k)
    with pytest.raises(SentioB200Error, match=r"rc=-4\).*too large"):
        pipe.engine.merge_shards_dev(*pipe._views(buf[0], B, k, 0), nbytes, G)
