"""CPU checks of tests/small_kernels_oracle.py, which the K3 / K4 / K6 edge tests on the GPU rely on:

* the merge oracle uses K1's total order on f64 scores (+0.0 above -0.0, which a ``-score`` sort key cannot express);
* ``mmr_vec`` / ``semantic_vec`` are bit-identical to ``oracle.scorers`` on dyadic inputs;
* the restated fusion oracle (with its mutant hooks switched off) equals ``oracle.fusion.fuse``;
* power: every seeded defect changes the expected output of at least one generated case.
"""
import numpy as np
import pytest

import small_kernels_oracle as so
from oracle import fusion, scorers


def test_merge_order_ranks_positive_zero_above_negative_zero():
    assert so.f64_key(0.0) > so.f64_key(-0.0) > so.f64_key(-1e-300)
    assert so.f64_key(1e-300) > so.f64_key(0.0)
    assert so.f64_key(-1.0) > so.f64_key(-2.0) and so.f64_key(2.0) > so.f64_key(1.0)
    # one shard holds -0.0 with the lower id, the other +0.0 with the higher id: +0.0 still comes first
    ids = np.asarray([[[5]], [[9]]], np.int64)
    sc = np.asarray([[[-0.0]], [[0.0]]])
    cnt = np.ones((2, 1), np.int32)
    got_ids, got_sc, got_cnt = so.merge_oracle((ids, sc, cnt), 2, 1)
    assert got_ids.tolist() == [[9]] and not np.signbit(got_sc[0, 0]) and got_cnt.tolist() == [1]
    # a plain (-score, id) key would have kept id 5
    assert sorted([(-(-0.0), 5), (-0.0, 9)])[0][1] == 5


def test_merge_oracle_on_a_hand_case():
    # shard 0: ids 1, 2 (count 2) + poison; shard 1: id 10 (count 1) + poison; k = 3
    ids = np.asarray([[[1, 2, 3]], [[10, 11, 12]]], np.int64)
    sc = np.asarray([[[0.5, 0.25, 1e300]], [[0.5, 1e300, 1e300]]])
    cnt = np.asarray([[2], [1]], np.int32)
    got = so.merge_oracle((ids, sc, cnt), 2, 3)
    assert got[0].tolist() == [[1, 10, 2]] and got[1].tolist() == [[0.5, 0.5, 0.25]] and got[2].tolist() == [3]
    got = so.merge_oracle((ids, sc, cnt), 2, 4)
    assert got[0].tolist() == [[1, 10, 2, -1]] and got[1].tolist() == [[0.5, 0.5, 0.25, 0.0]]


@pytest.mark.parametrize("n,d,lam,w", [(1, 3, 0.7, 0.5), (2, 7, 0.3, 0.5), (31, 16, 0.0, 0.5), (64, 7, 1.0, 0.5),
                                       (150, 24, 0.3, 0.0), (200, 33, 0.7, 0.5)])
@pytest.mark.parametrize("kind", ["mixed", "zero_query", "identical"])
def test_mmr_vec_bit_identical_to_reference_loop(n, d, lam, w, kind):
    q, C = so.mmr_case(n * 31 + d, n, d, kind)
    q64, c64 = q.astype(np.float64), [r.astype(np.float64) for r in C]
    want = np.asarray(scorers.mmr(q64, c64, lam, w))
    assert np.array_equal(so.mmr_vec(q, C, lam, w), want)
    assert np.array_equal(so.semantic_vec(q, C, w), np.asarray(scorers.semantic(q64, c64, w)))


def test_mmr_cases_contain_the_edges():
    q, C = so.mmr_case(1, 2049, 8)
    for a, off in ((0, 1), (3, 32), (5, 1024)):
        assert np.array_equal(C[a], C[a + off]) and (C[a] != 0).any()
    assert (C[2] == 0).all() and (C[-1] == 0).all()
    assert any(np.array_equal(r, -q) for r in C)   # anti-aligned with the query
    q, C = so.mmr_case(1, 40, 8, "identical")
    assert (C == C[0]).all() and C[0].sum() == 1.0


@pytest.mark.parametrize("method", ["rrf", "weighted_rrf", "comb_sum"])
def test_restated_fusion_equals_oracle(method):
    for seed in range(3):
        kw, _ = so.fuse_case(seed, method, rrf_k=(0.5, 1, 60)[seed])
        d, s, p, ex = kw["dense"], kw["sparse"], kw["plugin"], kw["extra"]
        for b in range(d[0].shape[0]):
            rows = [so._rows(x, b) for x in (d, s, p)]
            exb = [list(ex[b, e]) for e in range(ex.shape[1])]
            want = fusion.fuse(method, kw["rrf_k"], kw["w_dense"], kw["w_sparse"], *rows, kw["k"], exb)
            got = so._fuse_restated(method, kw["rrf_k"], kw["w_dense"], kw["w_sparse"], *rows, kw["k"], exb, None)
            assert got == want, (method, seed, b)


def test_fuse_cases_contain_the_edges():
    kw, (ids, sc, src, cnt) = so.fuse_case(0, "comb_sum")
    d_ids, d_sc, d_n = kw["dense"]
    assert d_n[1] == 0 and d_n[2] == 1
    assert (d_sc[3, :d_n[3]] == 0.5).all()
    past = np.arange(d_ids.shape[1])[None, :] >= d_n[:, None]
    assert past.any() and (d_sc[past] == so.POISON_SCORE).all()
    assert any(len(set(d_ids[b, :d_n[b]])) < d_n[b] for b in range(len(d_n)))      # duplicates inside a list
    p_ids, _, p_n = kw["plugin"]
    assert any(i >= 10_000 for b in range(len(p_n)) for i in p_ids[b, :p_n[b]])     # plugin-only ids
    assert (src[ids >= 10_000] == 0).all() and (ids[cnt[:, None] <= np.arange(ids.shape[1])[None, :]] == -1).all()


def _merge_mutant_cases():
    for seed, (G, B, k) in enumerate([(2, 9, 5), (3, 7, 16), (8, 5, 4)]):
        rec, want = so.merge_case(seed, G, B, k)
        yield rec, G, k, want


def _differs(a, b):
    return not all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("mutant", so.MERGE_MUTANTS)
def test_power_merge_mutants(mutant):
    assert any(_differs(so.merge_oracle(rec, G, k, mutant), want) for rec, G, k, want in _merge_mutant_cases())


@pytest.mark.parametrize("mutant", so.FUSE_MUTANTS)
def test_power_fuse_mutants(mutant):
    hits = 0
    for method in ("rrf", "weighted_rrf", "comb_sum"):
        kw, want = so.fuse_case(11, method)
        hits += _differs(so.fuse_oracle(**kw, mutant=mutant), want)
    assert hits


@pytest.mark.parametrize("mutant", so.MMR_MUTANTS)
def test_power_mmr_mutants(mutant):
    hits = 0
    for n, d, lam, w, kind in [(40, 7, 0.7, 0.5, "mixed"), (33, 5, 0.0, 0.5, "identical"), (40, 7, 1.0, 0.5, "mixed"),
                               (1100, 16, 0.3, 0.5, "mixed")]:
        q, C = so.mmr_case(n + d, n, d, kind)
        hits += not np.array_equal(so.mmr_vec(q, C, lam, w, mutant), so.mmr_vec(q, C, lam, w))
    assert hits
