"""Oracles and case generators for the small kernels every hybrid query passes through (TEST INFRASTRUCTURE):
K6 shard merge, K3 fusion and K4 semantic / MMR.

* ``merge_oracle``   -- union of every shard's first ``count`` entries, (score desc, id asc) in K1's total order on f64
                        scores (+0.0 ranks above -0.0), cut to k.
* ``fuse_oracle``    -- ``oracle.fusion.fuse`` over the ABI's array form (counts clipped to the stride, ``src`` bits,
                        -1 / 0.0 / 0 padding).
* ``mmr_vec``        -- vectorised ``oracle.scorers.mmr``: rel vector, Gram matrix ``C @ C.T`` and an incremental
                        max-redundancy, O(n^2) per pick instead of the reference loop's O(n^3).  On dyadic inputs
                        (``dyadic``) every fp64 dot product is exact, so it is bit-identical to the loop.
* ``*_case``         -- seeded generators returning (inputs, expected).  Entries past a list's count hold POISON: high
                        scores and plausible ids, so a kernel that reads past the count returns a wrong answer.

Every oracle takes ``mutant=``: a seeded defect (``MERGE_MUTANTS`` / ``FUSE_MUTANTS`` / ``MMR_MUTANTS``).
tests/test_small_kernels_oracle_cpu.py shows each defect changes the expected output of at least one generated case.
"""
from __future__ import annotations

import numpy as np

from oracle import fusion as fusion_oracle

MERGE_MUTANTS = ("ties_id_desc", "past_count")
FUSE_MUTANTS = ("rrf_rank_1_based", "comb_sum_first_wins", "extra_by_representative")
MMR_MUTANTS = ("ge_not_gt", "ties_to_highest_index", "redundancy_from_neg_inf", "no_clip")

POISON_SCORE = 1e300


# ------------------------------------------------------------------------------------------------------------ K6 merge
def f64_key(x: float) -> int:
    """K1's total order on f64 scores as an unsigned integer: larger key = better score; +0.0 above -0.0."""
    u = int(np.float64(x).view(np.uint64))
    return u ^ (0xFFFFFFFFFFFFFFFF if u >> 63 else 0x8000000000000000)


def merge_oracle(records, G: int, k: int, mutant: str | None = None):
    """records = (ids [G,B,k] i64, scores [G,B,k] f64, counts [G,B] i32) -> (ids [B,k], scores [B,k], counts [B])."""
    r_ids, r_sc, r_cnt = records
    B = r_ids.shape[1]
    ids = np.full((B, k), -1, np.int64)
    sc = np.zeros((B, k), np.float64)
    cnt = np.zeros(B, np.int32)
    for b in range(B):
        cand = []
        for g in range(G):
            n = k if mutant == "past_count" else int(r_cnt[g, b])
            cand += [(f64_key(r_sc[g, b, j]), int(r_ids[g, b, j]), float(r_sc[g, b, j])) for j in range(n)]
        if mutant == "ties_id_desc":
            cand.sort(key=lambda t: (-t[0], -t[1]))
        else:
            cand.sort(key=lambda t: (-t[0], t[1]))
        cand = cand[:k]
        cnt[b] = len(cand)
        ids[b, :len(cand)] = [c[1] for c in cand]
        sc[b, :len(cand)] = [c[2] for c in cand]
    return ids, sc, cnt


def merge_case(seed: int, G: int, B: int, k: int, scores=(1.0, 0.5, 0.25, 0.0, -0.0, -0.5, -2.0)):
    """Per-shard lists as K1 / K2 leave them: (score desc, id asc) in the total order, ids from disjoint per-shard ranges.
    Scores come from a small set, so exact ties straddle shard boundaries and rank k.  Counts: 0 for some (shard, query)
    pairs, below k, exactly k.  -> (records, expected)."""
    rng = np.random.default_rng(seed)
    span = 4 * k + 8
    r_ids = np.zeros((G, B, k), np.int64)
    r_sc = np.zeros((G, B, k), np.float64)
    r_cnt = np.zeros((G, B), np.int32)
    choices = np.asarray(scores, np.float64)
    for g in range(G):
        for b in range(B):
            c = (0, k, int(rng.integers(1, k + 1)), int(rng.integers(0, k + 1)))[(g + 3 * b) % 4]
            ids = rng.choice(span, size=k, replace=False).astype(np.int64) + g * span + 1000
            sc = choices[rng.integers(0, len(choices), size=k)]
            order = sorted(range(k), key=lambda j: (-f64_key(sc[j]), ids[j]))
            r_ids[g, b], r_sc[g, b] = ids[order], sc[order]
            r_cnt[g, b] = c
            # poison: high scores, plausible ids of this shard
            r_sc[g, b, c:] = POISON_SCORE
    records = (r_ids, r_sc, r_cnt)
    return records, merge_oracle(records, G, k)


# ------------------------------------------------------------------------------------------------------------ K3 fusion
def _fuse_restated(method, rrf_k, dense_weight, sparse_weight, dense, sparse, plugin, top_k, extras, mutant):
    """oracle.fusion.fuse with seeded defects; mutant=None is pinned equal to it."""
    fused: dict = {}

    def add(key, value):
        fused[key] = fused.get(key, 0.0) + value

    r0 = 1 if mutant == "rrf_rank_1_based" else 0
    if method in ("rrf", "weighted_rrf"):
        for lst, w in ((dense, dense_weight), (sparse, sparse_weight), (plugin, None)):
            w = 1.0 if (method == "rrf" or w is None) else float(w)
            for rank, (doc_id, _s) in enumerate(lst):
                add(doc_id, (1.0 / (rrf_k + rank + r0)) if lst is plugin else w * (1.0 / (rrf_k + rank + r0)))
    else:
        for lst, weight in ((dense, float(dense_weight)), (sparse, float(sparse_weight)), (plugin, 0.2)):
            raw = {}
            for doc_id, s in lst:
                if mutant == "comb_sum_first_wins" and doc_id in raw:
                    continue
                raw[doc_id] = float(s)
            for doc_id, ns in fusion_oracle._normalise(raw).items():
                add(doc_id, weight * ns)
    merged, seen = [], set()
    for doc_id, _ in list(dense) + list(sparse):
        if doc_id not in seen:
            seen.add(doc_id)
            merged.append(doc_id)
    if mutant == "extra_by_representative":
        # row index = first-occurrence slot in the dense ++ sparse concatenation instead of the merged position
        slot = {}
        for t, (doc_id, _) in enumerate(list(dense) + list(sparse)):
            slot.setdefault(doc_id, t)
        for scores in extras or []:
            for doc_id in merged:
                if slot[doc_id] < len(scores):
                    add(doc_id, float(scores[slot[doc_id]]))
    else:
        for scores in extras or []:
            for doc_id, s in zip(merged, scores):
                add(doc_id, float(s))
    ranked = sorted(fused.items(), key=lambda kv: kv[1], reverse=True)[:top_k]
    return [(doc_id, score, doc_id in seen) for doc_id, score in ranked]


def _rows(lst, b):
    if lst is None:
        return []
    i, s, c = lst
    n = min(int(c[b]), i.shape[1])
    return [(int(i[b, j]), float(s[b, j])) for j in range(n)]


def fuse_oracle(method, rrf_k, w_dense, w_sparse, k, dense=None, sparse=None, plugin=None, extra=None,
                mutant: str | None = None):
    """Array form of the fusion oracle, same arguments and outputs as ``B200Engine.fuse``."""
    B = next(x for x in (dense, sparse, plugin) if x is not None)[0].shape[0]
    ids = np.full((B, k), -1, np.int64)
    sc = np.zeros((B, k), np.float64)
    src = np.zeros((B, k), np.int32)
    cnt = np.zeros(B, np.int32)
    for b in range(B):
        d, s, p = _rows(dense, b), _rows(sparse, b), _rows(plugin, b)
        ex = [list(extra[b, e]) for e in range(extra.shape[1])] if extra is not None else None
        if mutant is None:
            out = fusion_oracle.fuse(method, rrf_k, w_dense, w_sparse, d, s, p, k, ex)
        else:
            out = _fuse_restated(method, rrf_k, w_dense, w_sparse, d, s, p, k, ex, mutant)
        d_set, s_set = {i for i, _ in d}, {i for i, _ in s}
        for j, (doc_id, score, _has) in enumerate(out):
            ids[b, j], sc[b, j] = doc_id, score
            src[b, j] = (1 if doc_id in d_set else 0) | (2 if doc_id in s_set else 0)
        cnt[b] = len(out)
    return ids, sc, src, cnt


def _fuse_list(rng, B, stride, pool, score_set, dup_rate, counts):
    """One [B, stride] list: ids drawn from ``pool`` with in-list duplicates, scores from ``score_set`` (descending, as
    the retrievers hand them over), poison past the count."""
    ids = np.zeros((B, stride), np.int64)
    sc = np.zeros((B, stride), np.float64)
    for b in range(B):
        base = rng.choice(pool, size=stride, replace=len(pool) < stride)
        dup = rng.random(stride) < dup_rate
        for j in np.nonzero(dup)[0]:
            if j > 0:
                base[j] = base[rng.integers(0, j)]   # duplicate of an earlier entry: a cache hit prepended twice
        ids[b] = base
        sc[b] = -np.sort(-np.asarray(score_set)[rng.integers(0, len(score_set), stride)])
        c = int(counts[b])
        if c < stride:
            ids[b, c:] = rng.choice(pool, size=stride - c)
            sc[b, c:] = POISON_SCORE
    return ids, sc, np.asarray(counts, np.int32)


def fuse_case(seed: int, method: str, B: int = 40, stride: int = 24, k: int = 30, rrf_k=60, w_dense=0.7,
              w_sparse=0.3, plugin: bool = True, n_extra: int = 2, e_stride: int | None = None,
              s_stride: int | None = None, p_stride: int | None = None):
    """Lists with in-list duplicates, ids shared between dense / sparse / plugin, plugin-only ids, scorer rows, small
    score sets (ties, all-equal lists, negative raw scores), count-0 and one-item lists.  -> (kwargs, expected)."""
    rng = np.random.default_rng(seed)
    s_stride = stride if s_stride is None else s_stride
    p_stride = stride if p_stride is None else p_stride
    pool = np.arange(3 * stride + 5, dtype=np.int64) + 7

    def counts(st):
        c = rng.integers(0, st + 1, B)
        c[0], c[1 % B], c[2 % B], c[3 % B] = st, 0, 1, st
        return c

    d = _fuse_list(rng, B, stride, pool, (0.9, 0.5, 0.5, 0.25, -0.75), 0.25, counts(stride))
    s = _fuse_list(rng, B, s_stride, pool, (12.0, 3.5, 3.5, 1.0, -2.0), 0.2, counts(s_stride))
    # query 3: every dense score equal (comb_sum normalises the list to 1.0)
    d[1][3 % B, :] = 0.5
    kw = dict(method=method, rrf_k=rrf_k, w_dense=w_dense, w_sparse=w_sparse, k=k, dense=d, sparse=s)
    if plugin:
        ppool = np.concatenate([pool, np.arange(10_000, 10_000 + stride, dtype=np.int64)])   # plus plugin-only ids
        kw["plugin"] = _fuse_list(rng, B, p_stride, ppool, (4.0, 2.0, 1.0), 0.15, counts(p_stride))
    if n_extra:
        e = 2 * stride if e_stride is None else e_stride
        kw["extra"] = np.round(rng.standard_normal((B, n_extra, e)) * 8) / 64
    return kw, fuse_oracle(**kw)


# ------------------------------------------------------------------------------------------------------------ K4 MMR
def dyadic(rng, shape, lo: int = -8, hi: int = 8) -> np.ndarray:
    """Values j/8, |j| <= 8: exact in fp16 / fp32, and every fp64 dot product of d <= 2^40 of them is exact."""
    return (rng.integers(lo, hi + 1, size=shape) / 8.0).astype(np.float32)


def semantic_vec(q, C, w: float) -> np.ndarray:
    """Vectorised ``oracle.scorers.semantic``."""
    q = np.asarray(q, np.float64)
    C = np.asarray(C, np.float64)
    qn = np.sqrt(q @ q)
    dn = np.sqrt(np.einsum("ij,ij->i", C, C))
    den = qn * dn
    out = np.zeros(len(C))
    ok = (qn > 0) & (dn > 0)
    out[ok] = (C[ok] @ q) / den[ok] * w
    return out


def mmr_prep(q, C):
    """(rel [n], cosine Gram matrix [n, n]) -- the O(n^2 d) part of ``mmr_vec``, reusable across lambda / weight."""
    q = np.asarray(q, np.float64)
    C = np.asarray(C, np.float64)
    n = len(C)
    qn = np.sqrt(q @ q)
    dn = np.sqrt(np.einsum("ij,ij->i", C, C))
    den = qn * dn
    rel = np.zeros(n)
    nz = den != 0
    rel[nz] = (C[nz] @ q) / den[nz]
    gden = dn[:, None] * dn[None, :]
    sim = np.zeros((n, n))
    np.divide(C @ C.T, gden, out=sim, where=gden != 0)
    return rel, sim


def mmr_vec(q, C, lambda_: float, weight: float, mutant: str | None = None, prep=None) -> np.ndarray:
    """Vectorised ``oracle.scorers.mmr`` (rel vector, Gram matrix, incremental max-redundancy); ``prep`` = mmr_prep(q, C)."""
    n = len(C)
    if n == 0:
        return np.zeros(0)
    rel, sim = mmr_prep(q, C) if prep is None else prep
    sim = np.ascontiguousarray(sim.T)   # row idx = column idx of the (symmetric) Gram matrix, read contiguously
    red = np.full(n, -np.inf) if mutant == "redundancy_from_neg_inf" else np.zeros(n)
    scores = np.zeros(n)
    selected = np.zeros(n, bool)
    oml = 1 - lambda_
    for _ in range(n):
        with np.errstate(invalid="ignore"):   # 0 * -inf of the redundancy_from_neg_inf mutant
            val = lambda_ * rel - oml * red
        cand = np.nonzero(~selected)[0]
        v = val[cand]
        if mutant == "ge_not_gt":
            ok = cand[v >= -1.0]
            if len(ok) == 0:
                break
            vm = val[ok].max()
            idx = int(ok[np.nonzero(val[ok] == vm)[0][-1]])
        else:
            ok = cand[v > -1.0]
            if len(ok) == 0:
                break
            vm = val[ok].max()
            hit = ok[np.nonzero(val[ok] == vm)[0]]
            idx = int(hit[-1] if mutant == "ties_to_highest_index" else hit[0])
        best = val[idx]
        selected[idx] = True
        scores[idx] = best * weight
        col = sim[idx]
        red = np.where(col > red, col, red)   # Python max(redundancy, cos): keeps the left operand unless cos is larger
    fill = scores == 0.0
    scores[fill] = rel[fill] * weight * lambda_
    if mutant == "no_clip":
        return scores
    return np.where(scores > 0.0, scores, 0.0)


def mmr_case(seed: int, n: int, d: int, kind: str = "mixed"):
    """Dyadic (q, C).  kind "mixed": exact duplicate candidates at i / i+1 (same warp), i / i+32 (different warps) and
    i / i+1024 (same thread, next ``sel_mask`` slot), zero-norm candidates and anti-aligned candidates (negated query:
    the clip path).  kind "zero_query": the same with q = 0.  kind "identical": every candidate the same unit vector."""
    rng = np.random.default_rng(seed)
    q = dyadic(rng, d)
    C = dyadic(rng, (n, d))
    if kind == "identical":
        e = np.zeros(d, np.float32)
        e[int(rng.integers(0, d))] = 1.0
        return q, np.tile(e, (n, 1))
    for a, off in ((0, 1), (3, 32), (5, 1024), (n // 2, 1), (n // 3, 32)):
        if a + off < n:
            # close to the query, so the pair competes for an early pick while both members are unselected
            C[a] = q
            C[a, rng.integers(0, d, size=max(1, d // 8))] = dyadic(rng, max(1, d // 8))
            C[a + off] = C[a]
    for z in (2, n - 1, n // 4):
        if 0 <= z < n and n > 1:
            C[z] = 0.0
    for j in range(min(n, 6, max(1, n // 8))):
        i = (7 + 13 * j) % n
        if not (C[i] == 0).all():
            C[i] = -q if (q != 0).any() else C[i]
    if kind == "zero_query":
        q = np.zeros(d, np.float32)
    return q, C
