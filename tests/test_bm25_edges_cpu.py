"""CPU checks of tests/bm25_edges.py, which tests/test_bm25_edges_gpu.py relies on:

* without a defect, the kernel model equals FastBM25 bit for bit and its top-k equals the rank_bm25 order;
* the sample-bound model shows each path case reaches its path (more than 12288 candidates, a tight bound);
* power: every seeded defect changes the expected output (ids, counts or score bits) of at least one GPU case.
"""
import numpy as np
import pytest

import bm25_edges as be


def _differs(case, defect, rows=None):
    want = be.model_topk(case, None, rows)[0]
    return any(not all(np.array_equal(x, y) for x, y in zip(got, want)) for got in be.model_topk(case, defect, rows))


def _cases_small():
    for v in ("okapi", "plus"):
        yield be.range_edge_case(513, v)
        yield be.range_edge_case(4 * be.RANGE + 1, v)
        yield be.head_case(4096, v)
        yield be.many_heads_case(v)
        yield be.straddle_case(v)
        yield be.extreme_case("b_1", v)
    for kind in ("empty_sampled", "exact_ks", "tight"):
        yield be.sample_case(kind)
    yield be.extreme_case("negative_floor")
    yield be.extreme_case("idf_zero")


@pytest.mark.parametrize("case", list(_cases_small()), ids=lambda c: c.name)
def test_model_without_defect_is_fastbm25_and_rank_bm25_order(case):
    f = be.fast(case.idx)
    want_rows = []
    for terms in case.queries:
        s = f.get_scores(list(terms))
        assert np.array_equal(be.bits(be.model_scores(case.idx, terms)), be.bits(s))
        want_rows.append(be.ref_topk(s, case.k))
    ids, sc, cnt = be.padded(want_rows, [f.get_scores(list(t)) for t in case.queries], case.k, case.id_base)
    got = be.model_topk(case)
    assert len(got) == 1
    assert np.array_equal(got[0][0], ids) and np.array_equal(got[0][1], be.bits(sc)) and np.array_equal(got[0][2], cnt)


def test_edge_positions_cover_every_boundary():
    n = 3 * be.RANGE + 1
    p = set(be.edge_positions(n).tolist())
    assert {0, 1, n - 1, 511, 512, 513, be.RANGE - 1, be.RANGE, be.RANGE + 1, 3 * be.RANGE - 1, 3 * be.RANGE} <= p
    assert be.edge_positions(1).tolist() == [0]


def test_sample_bound_model_on_hand_cases():
    s = np.zeros(4 * be.RANGE)
    s[[3, 9000, 17000, 30000]] = [5.0, 4.0, 3.0, 2.0]
    assert be.sample_bound(s, 4) == 2.0                  # one per range, exact values on a bucket edge
    assert be.sample_bound(s, 5) == 5e-324               # ceil(5/4) = 2 > one positive per range: every positive
    s[1] = 1.0 + 2.0 ** -30                              # below the 12 mantissa bits the bucket keeps
    assert be.sample_bound(s[:be.RANGE], 2) == 1.0
    assert be.sample_bound(np.array([0.5, -1.0, 0.0]), 1) == 0.5   # one range: S = 1


@pytest.mark.parametrize("m", [12287, 12288, 12289, 40000])
def test_tie_cases_make_m_candidates(m):
    case = be.tie_case(m, "okapi")
    s = be.fast(case.idx).get_scores(list(case.queries[0]))
    assert len(be.candidates(s, case.k)) == m
    assert (len(be.candidates(s, case.k)) > be.STAGE) == (m > be.STAGE)


def test_both_ends_case_exceeds_the_stage_and_wins_at_both_ends():
    case = be.both_ends_case("okapi")
    s = be.fast(case.idx).get_scores(list(case.queries[0]))
    assert len(be.candidates(s, case.k)) > be.STAGE
    top = be.ref_topk(s, case.k)
    assert {0, 9, case.idx.n_docs - 1, case.idx.n_docs - 10} <= set(top[:20].tolist())


def test_sample_cases_reach_their_paths():
    for kind in ("empty_sampled", "exact_ks"):
        s = be.fast(be.sample_case(kind).idx).get_scores(list(be.sample_case(kind).queries[0]))
        assert be.sample_bound(s, 10) == 5e-324 if kind == "empty_sampled" else be.sample_bound(s, 10) > 5e-324
        top = be.ref_topk(s, 10)
        assert (top >= 4 * be.RANGE).all()               # the true top k lies in range 4, which is not sampled
    s = be.fast(be.sample_case("tight").idx).get_scores(list(be.sample_case("tight").queries[0]))
    assert len(be.candidates(s, 10)) == 12 and len(be.candidates(s, 10, floor=True)) == 8


def test_strip_case_has_several_sub_batches_and_multi_range_ctas():
    case = be.strip_case("okapi")
    n, B = case.idx.n_docs, len(case.queries)
    sbq = be.sub_batch_size(n, B)
    assert sbq < B and -(-B // sbq) >= 3
    for b0 in range(0, B, sbq):
        assert be.ranges_per_cta(132, min(sbq, B - b0), n) > 1


# defect -> cases whose expected output it must change (any one of them suffices)
POWER = {
    "first_of_sub": lambda: [be.range_edge_case(4 * be.RANGE + 1, "okapi")],
    "last_of_sub": lambda: [be.range_edge_case(4 * be.RANGE + 1, "okapi")],
    "short_last_range": lambda: [be.range_edge_case(4 * be.RANGE + 1, "plus")],
    "reverse_terms": lambda: [be.long_query_case("okapi")],
    "drop_after_512": lambda: [be.long_query_case("okapi")],
    "dup_once": lambda: [be.range_edge_case(513, "okapi")],
    "plus_head_no_delta": lambda: [be.head_case(4096, "plus")],
    "head_row_alias": lambda: [be.many_heads_case("okapi")],
    "sample_floor": lambda: [be.sample_case("tight")],
    "ties_desc": lambda: [be.straddle_case("okapi")],
    "stage_only": lambda: [be.both_ends_case("okapi")],
    "sub_batch_0": lambda: [be.strip_case("okapi")],
    "no_id_base": lambda: [be.straddle_case("okapi")],
}


def test_power_table_covers_every_defect():
    assert set(POWER) == set(be.DEFECTS)


@pytest.mark.parametrize("defect", be.DEFECTS)
def test_power_defect_changes_a_gpu_case(defect):
    hits = []
    for case in POWER[defect]():
        rows = case.rows
        if defect == "sub_batch_0":
            sbq = be.sub_batch_size(case.idx.n_docs, len(case.queries))
            rows = [sbq, 2 * sbq]
        elif len(case.queries) > 4 and rows is None and case.idx.n_docs * len(case.queries) > 10**6:
            rows = list(range(len(case.queries)))
        hits.append(_differs(case, defect, rows))
    assert any(hits), defect
