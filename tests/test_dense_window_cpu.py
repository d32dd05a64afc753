"""The adversarial window corpora of tests/window_oracle.py, checked on the CPU: for every case and scan the exact top-k
differs from the approximate top-k (a), the true eps keeps every exact top-k row inside the window (b), and every
mutant the case targets -- an eps or a window too narrow by one term -- leaves an exact top-k row outside it (c).
Every approximate key may sit anywhere within the accumulation part of eps of its emulated value."""
import numpy as np
import pytest

import window_oracle as wo

MUTANT_SCANS = {"M7": ("mma",)}   # the sampling pass exists on the wgmma scan only


@pytest.fixture(scope="module", params=sorted(wo.CASES))
def case(request):
    return wo.adversarial_case(request.param)


def _scans(case):
    return [(scan, scan == "mma") for scan in case.scans]


def test_exact_top_k_is_the_decoys_and_the_window_keeps_them(case):
    slot = wo.make_slot(case.x, case.storage, case.metric)
    for scan, mma in _scans(case):
        for m in range(wo.N_ADV):
            v = wo.analyse(slot, case.q[m], case.k, mma, case.bounds, match=case.match)
            decoys, baits = case.bands[m]
            assert sorted(v.exact_top.tolist()) == sorted(decoys.tolist()), f"{case.name} {scan} q {m}: exact top-k"
            assert v.approx_differs, f"{case.name} {scan} q {m}: (a) the approximate top-k must differ"
            assert v.kept, f"{case.name} {scan} q {m}: (b) margin {v.margin_kept:.3f} eps"


def test_each_targeted_mutant_drops_an_exact_row(case):
    slot = wo.make_slot(case.x, case.storage, case.metric)
    for mutant in case.mutants + (("M2",) if case.storage == "float16" else ()):
        for scan, mma in _scans(case):
            if scan not in MUTANT_SCANS.get(mutant, (scan,)):
                continue
            margins = [wo.analyse(slot, case.q[m], case.k, mma, case.bounds, mutant=mutant,
                                  b_mut=case.bounds0 if mutant == "M6" else None, match=case.match).margin_missed
                       for m in range(wo.N_ADV)]
            assert max(margins) > 0, f"{case.name} {scan} {mutant}: (c) margins {margins}"


def test_upsert_cases_raise_the_bounds(case):
    if case.x0 is None:
        pytest.skip("not an upsert case")
    b0, b = case.bounds0, case.bounds
    if case.storage == "float32":
        assert b0.sigma < 1e-9 < b.sigma
    else:
        assert b.rho > 10 * b0.rho


def test_euclid_cases_stay_on_the_scans(case):
    """The Euclid queries pass the fp64-resolution routing rule: no brute force up front."""
    if case.metric != "euclid":
        pytest.skip("Euclid only")
    for m in range(wo.N_ADV):
        for _, mma in _scans(case):
            eps = wo.query_eps(case.q[m], wo.D, case.storage, "euclid", mma, case.bounds)
            assert wo.euclid_resolves(case.q[m], case.bounds, eps)


def test_filtered_case_has_more_than_2048_matches_and_higher_rows_outside_the_filter():
    case = wo.adversarial_case("filtered_f32_cosine")
    assert case.match.sum() > 2048
    s = wo.exact_keys(wo.make_slot(case.x, case.storage, case.metric), case.q[0])
    decoys, baits = case.bands[0]
    assert (s[~case.match] > s[decoys].max()).sum() >= 2 * case.k


def test_eps_restatement_terms():
    """An exactly representable query has no rounding term; a rounded one adds ||fp16(q^) - q^|| (1.0001)."""
    q = np.zeros(wo.D, np.float32)
    q[:4] = 1.0
    assert wo.query_eps(q, 64, "float16", "cosine", True, wo.Bounds()) == wo.eps_mma_acc(64)
    assert wo.query_eps(q, 64, "float16", "cosine", False, wo.Bounds()) == wo.eps_fp32(64)
    q[:4] = [0.3, 0.7, 0.9, 0.11]
    t = wo.prep_query(q, 64)[2]
    assert t > 0
    e = wo.query_eps(q, 64, "float16", "cosine", True, wo.Bounds())
    assert abs(e - (np.sqrt(t) * 1.0001 + wo.eps_mma_acc(64))) < 1e-9
    b = wo.Bounds(rho=1e3, hmax=5e5, sigma=1e-4)
    assert wo.query_eps(q, 64, "float32", "dot", True, b) > 1e3 * e
    assert wo.query_eps(q, 64, "float32", "dot", True, b, mutant="M3") < 2 * e + 1e-4
    assert wo.query_eps(q * 100, 64, "float16", "euclid", True, b, mutant="M4") < \
        wo.query_eps(q * 100, 64, "float16", "euclid", True, b) / 10


def test_select_bound_restatement():
    """The radix select's bound is the k-th largest key when its bucket stays crowded, lower when it stops early."""
    rng = np.random.default_rng(1)
    a = (0.5 + 1e-4 * rng.standard_normal(300)).astype(np.float32)
    rows = np.arange(300)
    lb = wo.select_lb(a, rows, 100)
    kth = np.sort(a)[::-1][99]
    assert lb <= kth and kth - lb < 1e-5
    a2 = np.concatenate([np.float32([0.9] * 100), np.float32([0.1] * 5)])
    assert wo.select_lb(a2, np.arange(105), 100) <= 0.9


def test_crowded_rows_overflow_one_list_of_each_scan():
    x, q, rows = wo.crowded_case()
    assert len(x) == wo.CROWD_N
    tiles = (rows // 128) % wo.NUM_SMS
    assert (tiles == 0).sum() > wo.mma_list_capacity(wo.CROWD_N, 10), "wgmma CTA 0's survivor list overflows"
    core_cta = (rows // 32) % wo.NUM_SMS
    assert (core_cta == 0).sum() > 128, "CUDA-core CTA 0's 128-entry list is all window rows"
    slot = wo.make_slot(x, "float16", "cosine")
    for m in range(wo.N_ADV):
        s = wo.exact_keys(slot, q[m])
        assert set(np.argsort(-s, kind="stable")[:10].tolist()) <= set(rows.tolist())
