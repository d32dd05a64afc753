"""K4 semantic / MMR scorer signals at their edges.

With dyadic inputs every fp64 dot product is exact, so the only roundings left are the IEEE-correct fp64 sqrt,
division and the `_rn` products, and the kernel must equal the oracle BIT FOR BIT (np.array_equal): n up to the 4096
limit (a thread owns up to 4 candidates, the `sel_mask` slots), exact duplicates inside a warp / across warps / in the
same thread's next slot (first index wins), zero-norm candidates, a zero query, lambda in {0, 0.3, 1}, w in {0, 0.5},
anti-aligned candidates (the clip at 0) and the early `break` (lambda = 0 over identical candidates)."""
import numpy as np
import pytest

import small_kernels_oracle as so

pytestmark = pytest.mark.gpu

SHAPES = [(n, d) for n in (1, 2, 31, 1023, 1024, 1025) for d in (1, 7, 384, 1024)] + \
         [(2049, 7), (2049, 1024), (4096, 1), (4096, 384)]
LAMBDA_W = [(0.0, 0.5), (0.3, 0.5), (1.0, 0.5), (0.3, 0.0)]


@pytest.fixture(scope="module")
def eng(built_lib):
    """An engine of its own: the stored-corpus tests load both dense slots."""
    from sentio_b200.engine import B200Engine

    e = B200Engine(0)
    yield e
    e.close()


def _check(eng, q, C, cases, what):
    prep = so.mmr_prep(q, C)
    for lam, w in cases:
        sem, mmr = eng.semantic_mmr(q, cand=C, w_sem=w, lambda_=lam, w_mmr=w)
        assert np.array_equal(sem, so.semantic_vec(q, C, w)), (what, lam, w)
        assert np.array_equal(mmr, so.mmr_vec(q, C, lam, w, prep=prep)), (what, lam, w)


@pytest.mark.parametrize("n,d", SHAPES)
def test_dyadic_bit_exact(eng, n, d):
    q, C = so.mmr_case(7 * n + d, n, d)
    _check(eng, q, C, LAMBDA_W, (n, d))


@pytest.mark.parametrize("n,d", [(31, 7), (1025, 384), (4096, 7)])
def test_zero_query(eng, n, d):
    q, C = so.mmr_case(n + d, n, d, "zero_query")
    _check(eng, q, C, LAMBDA_W, (n, d))


@pytest.mark.parametrize("n", [2, 33, 1025, 2049])
def test_identical_candidates_lambda_zero_breaks_early(eng, n):
    """lambda = 0: after the first pick every value is -1.0, which the strict `>` from -1.0 never takes -> break."""
    q, C = so.mmr_case(n, n, 16, "identical")
    rel, sim = so.mmr_prep(q, C)
    assert (sim == 1.0).all()
    _check(eng, q, C, [(0.0, 0.5), (0.3, 0.5), (1.0, 0.5)], n)


def test_duplicate_pairs_first_index_wins(eng):
    """A pair of duplicates close to the query at i / i+1, i / i+32 and i / i+1024: the pick order inside each pair is
    visible in the output (the first pick scores lambda*rel, its twin pays the redundancy)."""
    n, d = 2049, 64
    q, C = so.mmr_case(3, n, d)
    lam, w = 0.7, 0.5
    want = so.mmr_vec(q, C, lam, w)
    for a, off in ((0, 1), (3, 32), (5, 1024)):
        assert want[a] != want[a + off]
    for mutant in ("ge_not_gt", "ties_to_highest_index"):
        assert not np.array_equal(so.mmr_vec(q, C, lam, w, mutant), want)
    _check(eng, q, C, [(lam, w)], "pairs")


@pytest.mark.parametrize("n", [5, 1500])
def test_sem_only_and_mmr_only_equal_the_combined_call(eng, n):
    """retrievers/scorers.py asks for one signal at a time."""
    q, C = so.mmr_case(n, n, 48)
    sem, mmr = eng.semantic_mmr(q, cand=C, w_sem=0.5, lambda_=0.3, w_mmr=0.5)
    sem1, none1 = eng.semantic_mmr(q, cand=C, w_sem=0.5, lambda_=0.3, w_mmr=0.5, want_mmr=False)
    none2, mmr2 = eng.semantic_mmr(q, cand=C, w_sem=0.5, lambda_=0.3, w_mmr=0.5, want_sem=False)
    assert none1 is None and none2 is None
    assert np.array_equal(sem1, sem) and np.array_equal(mmr2, mmr)


@pytest.mark.parametrize("storage", ["float16", "float32"])
def test_candidates_by_id_from_a_stored_slot(eng, storage):
    """cand_ids gather the slot's rows (fp16 rows, or a float32 slot's input rows); ids outside the slot gather a zero
    vector, which then scores like a zero-norm candidate."""
    rng = np.random.default_rng(21)
    n_rows, d, base = 3000, 96, 500
    x = so.dyadic(rng, (n_rows, d))
    x[17] = 0.0
    slot = 0 if storage == "float16" else 1
    eng.load_dense(x.astype(np.float16) if storage == "float16" else x, id_base=base, slot=slot, storage=storage)
    ids = rng.integers(base, base + n_rows, 1100).astype(np.int64)
    ids[[3, 4, 1027]] = ids[2]                                    # duplicates: same warp, next slot
    ids[[10, 11, 12, 13, 14]] = [base - 1, base + n_rows, -5, 0, base + n_rows + 10 ** 6]   # outside the slot
    ids[20] = base + 17                                           # a stored zero row
    q = so.dyadic(rng, d)
    C = np.zeros((len(ids), d), np.float32)
    inside = (ids >= base) & (ids < base + n_rows)
    C[inside] = x[ids[inside] - base]
    prep = so.mmr_prep(q, C)
    for lam, w in [(0.3, 0.5), (1.0, 0.5), (0.0, 0.5)]:
        sem, mmr = eng.semantic_mmr(q, cand_ids=ids, w_sem=w, lambda_=lam, w_mmr=w, slot=slot)
        assert np.array_equal(sem, so.semantic_vec(q, C, w)), (storage, lam)
        assert np.array_equal(mmr, so.mmr_vec(q, C, lam, w, prep=prep)), (storage, lam)
        assert (sem[10:15] == 0.0).all()


def test_more_than_4096_candidates_is_unsupported(eng):
    from sentio_b200._lib import SentioB200Error

    rng = np.random.default_rng(0)
    with pytest.raises(SentioB200Error, match=r"rc=-4\).*4096"):
        eng.semantic_mmr(so.dyadic(rng, 8), cand=so.dyadic(rng, (4097, 8)), w_sem=0.5, lambda_=0.3, w_mmr=0.5)


def test_gaussian_2048_candidates(eng):
    rng = np.random.default_rng(8)
    n, d = 2048, 384
    C = rng.standard_normal((n, d)).astype(np.float32)
    C[100:140] = C[0:40] + 0.05 * rng.standard_normal((40, d)).astype(np.float32)   # near duplicates
    q = rng.standard_normal(d).astype(np.float32)
    sem, mmr = eng.semantic_mmr(q, cand=C, w_sem=0.8, lambda_=0.5, w_mmr=0.5)
    assert np.allclose(sem, so.semantic_vec(q, C, 0.8), rtol=1e-9, atol=1e-12)
    assert np.allclose(mmr, so.mmr_vec(q, C, 0.5, 0.5), rtol=1e-9, atol=1e-12)
