"""K3 fusion at its edges == oracle/fusion.fuse bit for bit: duplicates inside one list (cache hits prepended to the
dense list -- comb_sum's last-wins path), a plugin list overlapping both lists plus plugin-only ids, scorer rows with
e_stride below / equal to / above the merged count, all-equal / negative / one-item / count-0 lists, rrf_k in
{0.5, 1, 60}, k = 1 and k above the number of unique ids, M = 4096 candidates per query, and the device entry point
with d_stride != s_stride != k.  Entries past every count hold poison (tests/small_kernels_oracle.py)."""
import numpy as np
import pytest

import small_kernels_oracle as so

pytestmark = pytest.mark.gpu

METHODS = ["rrf", "weighted_rrf", "comb_sum"]


def _assert_same(got, want, what):
    ids, sc, src, cnt = got
    w_ids, w_sc, w_src, w_cnt = want
    assert np.array_equal(cnt, w_cnt), what
    assert np.array_equal(ids, w_ids), what
    assert np.array_equal(np.asarray(sc, np.float64).view(np.uint64), w_sc.view(np.uint64)), what
    assert np.array_equal(src, w_src), what


def _run(engine, kw):
    kw = dict(kw)
    return engine.fuse(kw.pop("method"), kw.pop("rrf_k"), kw.pop("w_dense"), kw.pop("w_sparse"), kw.pop("k"), **kw)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("rrf_k", [0.5, 1, 60])
def test_duplicates_plugin_and_scorer_rows(engine, method, rrf_k):
    for n_extra, e_stride in [(1, 5), (2, 24), (3, 60)]:
        kw, want = so.fuse_case(int(rrf_k * 10) + n_extra, method, B=300, stride=24, k=30, rrf_k=rrf_k,
                                n_extra=n_extra, e_stride=e_stride)
        _assert_same(_run(engine, kw), want, (method, rrf_k, n_extra, e_stride))


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("k", [1, 200])
def test_k_one_and_k_above_unique_ids(engine, method, k):
    """k = 200 exceeds the 3 * 24 candidates of a query: the tail is -1 / 0.0 / src 0 and the count is the number of
    unique ids."""
    kw, want = so.fuse_case(77 + k, method, B=64, stride=24, k=k)
    got = _run(engine, kw)
    _assert_same(got, want, (method, k))
    if k == 200:
        assert (got[3] < k).all()


@pytest.mark.parametrize("method", METHODS)
def test_without_plugin_or_scorer_rows(engine, method):
    kw, want = so.fuse_case(5, method, B=97, stride=40, k=50, plugin=False, n_extra=0)
    _assert_same(_run(engine, kw), want, method)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("strides", [(2048, 2048, None), (1366, 1365, 1365)])
def test_4096_candidates_per_query(engine, method, strides):
    d, s, p = strides
    kw, want = so.fuse_case(4096 + d, method, B=5, stride=d, s_stride=s, p_stride=p or 1, k=1000,
                            plugin=p is not None, n_extra=1, e_stride=300)
    _assert_same(_run(engine, kw), want, (method, strides))


def test_4097_candidates_per_query_is_unsupported(engine):
    from sentio_b200._lib import SentioB200Error

    kw, _ = so.fuse_case(1, "rrf", B=2, stride=2049, s_stride=2048, k=10, plugin=False, n_extra=0)
    with pytest.raises(SentioB200Error, match=r"rc=-4\).*4096"):
        _run(engine, kw)


@pytest.mark.parametrize("method", METHODS)
def test_device_entry_with_unequal_strides(engine, method):
    """sb_fuse_dev (what the pipeline calls) with d_stride = 24, s_stride = 17 and k = 30."""
    import torch

    kw, want = so.fuse_case(31, method, B=301, stride=24, s_stride=17, k=30, plugin=False, n_extra=0)
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in kw[n]) for n in ("dense", "sparse")]
    out = engine.fuse_dev(method, kw["rrf_k"], kw["w_dense"], kw["w_sparse"], kw["k"], dev[0], dev[1])
    torch.cuda.synchronize()
    _assert_same(tuple(t.cpu().numpy() for t in out), want, method)
