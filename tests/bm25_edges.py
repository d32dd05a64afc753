"""Corpus builders, references and a CPU model of K2 (BM25, ``sentio_b200/csrc/bm25.cu``) for its edge tests
(TEST INFRASTRUCTURE).

* ``index_from_triples`` -- a corpus given as explicit (doc, term, tf) postings plus filler tokens, so a case decides which
  docs hold which term, with which tf and which doc length.  Raw term ids; queries go through ``idx.term_ids``.
* ``ref_topk``           -- the rank_bm25 order the kernel must reproduce: stable ``argsort(-s)``, cut to k, keep ``> 0``.
* ``sample_bound``       -- the kernel's safe threshold: S = min(4, n_ranges) ranges starting at ``y * n_ranges // S``
                            each report the ceil(k/S)-th best positive score truncated to the lower edge of its 24-bit key
                            bucket ("every positive" when the range has fewer positives); the threshold is the minimum.
* ``model_scores`` / ``model_topk`` -- the same arithmetic as ``FastBM25`` and the same sample / collect / select /
  sub-batch structure as the kernel, with seeded defects (``DEFECTS``).  Without a defect they equal ``FastBM25`` and
  ``ref_topk``; tests/test_bm25_edges_cpu.py shows every defect changes the expected output of at least one case.
* ``*_case``             -- the inputs of tests/test_bm25_edges_gpu.py (cached), shared with the CPU power check.

Scores are compared through ``view(np.uint64)``: ``np.array_equal`` calls -0.0 and +0.0 equal.
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field

import numpy as np

from oracle.rank_bm25_port import FastBM25
from sentio_b200.index import build_bm25_from_token_ids

RANGE, SUB, STAGE, MAX_ROWS = 8192, 512, 12288, 64   # kRange, kSub, kBmStage, dense-row cap of bm25.cu
SMEM_FIXED, SMEM_PER_TERM = 8192 * 8 + 16 * 8 + 256 * 4 + 16, 88   # per-CTA shared memory of bm25_range_kernel
FILL = 1 << 24           # filler tokens: raw id FILL + doc (unique per doc, never queried)
UNKNOWN = (1 << 30)      # a raw token no corpus holds

DEFECTS = ("first_of_sub", "last_of_sub", "short_last_range", "reverse_terms", "drop_after_512", "dup_once",
           "plus_head_no_delta", "head_row_alias", "sample_floor", "ties_desc", "stage_only", "sub_batch_0",
           "no_id_base")


# ----------------------------------------------------------------------------------------------------------- corpora
def index_from_triples(n, doc, term, tf, fill=None, variant="okapi", **kw):
    """Doc d holds term[i] tf[i] times for every i with doc[i] == d, then ``fill[d]`` filler tokens (default 1)."""
    doc = np.asarray(doc, np.int64)
    term = np.asarray(term, np.int64)
    tf = np.broadcast_to(np.asarray(tf, np.int64), doc.shape)
    fill = np.ones(n, np.int64) if fill is None else np.broadcast_to(np.asarray(fill, np.int64), (n,))
    d_all = np.concatenate([np.repeat(doc, tf), np.repeat(np.arange(n, dtype=np.int64), fill)])
    t_all = np.concatenate([np.repeat(term, tf), FILL + np.repeat(np.arange(n, dtype=np.int64), fill)])
    o = np.argsort(d_all, kind="stable")
    off = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(d_all, minlength=n), out=off[1:])
    return build_bm25_from_token_ids(t_all[o], off, variant=variant, **kw)


def fast(idx) -> FastBM25:
    if "fast" not in idx.extras:
        idx.extras["fast"] = FastBM25(idx.indptr, idx.post_doc, idx.post_tf, idx.doc_len, idx.idf, idx.avgdl,
                                      idx.variant, k1=idx.k1, b=idx.b, delta=idx.delta)
    return idx.extras["fast"]


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)


def ref_topk(scores, k):
    order = np.argsort(-scores, kind="stable")[:k]
    return order[scores[order] > 0]


def padded(orders, scores_list, k, id_base=0):
    """Rows of ``ref_topk`` in the kernel's output layout: ids + id_base / -1, scores / 0.0, counts."""
    B = len(orders)
    ids = np.full((B, k), -1, np.int64)
    sc = np.zeros((B, k))
    cnt = np.zeros(B, np.int32)
    for b, (o, s) in enumerate(zip(orders, scores_list)):
        ids[b, :len(o)] = o + id_base
        sc[b, :len(o)] = s[o]
        cnt[b] = len(o)
    return ids, sc, cnt


def sub_batch_size(n_docs, B, blocked=False):
    """Queries per sub-batch of bm25_topk_enqueue (candidate lists, plus the carried scores of a long query)."""
    return max(1, min((1536 << 20) // (n_docs * (20 if blocked else 12) + 1), B))


def ranges_per_cta(num_sms, nq, n_docs):
    n_ranges = -(-n_docs // RANGE)
    return max(1, min(32, nq * n_ranges // (num_sms * 4)))


def max_term_block(smem_optin):
    """An upper bound of the kernel's term block (its static shared memory only lowers it)."""
    return (smem_optin - SMEM_FIXED) // SMEM_PER_TERM


def head_terms(idx):
    """Term -> dense-row rank (df desc, term asc) of every head term; rank >= MAX_ROWS has no row."""
    n = idx.n_docs
    if n < 4096:
        return {}
    df = np.diff(idx.indptr)
    heavy = np.flatnonzero(df * 4 >= n)
    heavy = heavy[np.lexsort((heavy, -df[heavy]))]
    return {int(t): r for r, t in enumerate(heavy)}


# ----------------------------------------------------------------------------------------------------------- model
def model_scores(idx, terms, defect=None):
    """FastBM25's arithmetic term by term in query order, with the seeded scoring defects."""
    n, V = idx.n_docs, idx.n_terms
    f = fast(idx)
    terms = [int(t) for t in terms]
    if defect == "reverse_terms":
        terms = terms[::-1]
    elif defect == "drop_after_512":
        terms = terms[:512]
    elif defect == "dup_once":
        terms = list(dict.fromkeys(terms))
    head = head_terms(idx) if defect in ("plus_head_no_delta", "head_row_alias") else {}
    slot0 = next((t for t, r in head.items() if r == 0), None)
    score = np.zeros(n)
    for t in terms:
        if t < 0 or t >= V:
            continue
        idf = float(f.idf[t])
        if idf == 0.0:
            continue
        src = slot0 if defect == "head_row_alias" and head.get(t, -1) >= MAX_ROWS else t
        lo, hi = f.indptr[src], f.indptr[src + 1]
        docs, tf = f.post_doc[lo:hi], f.post_tf[lo:hi]
        keep = np.ones(len(docs), bool)
        if defect == "first_of_sub":
            keep = docs % SUB != 0
        elif defect == "last_of_sub":
            keep = (docs % SUB != SUB - 1) & (docs != n - 1)
        docs, tf = docs[keep], tf[keep]
        if f.variant == "plus":
            absent = 0.0 if defect == "plus_head_no_delta" and t in head else idf * (f.delta + 0.0)
            contrib = np.full(n, absent)
            contrib[docs] = idf * (f.delta + (tf * (f.k1 + 1)) / (f.dnorm[docs] + tf))
            score += contrib
        else:
            score[docs] += idf * (tf * (f.k1 + 1) / (tf + f.dnorm[docs]))
    if defect == "short_last_range" and n % RANGE:
        score[n - n % RANGE:] = 0.0
    return score


def sample_bound(scores, k, floor=False):
    """The kernel's per-query threshold (see the module docstring); a double, 5e-324 = every positive score."""
    n = len(scores)
    n_ranges = -(-n // RANGE)
    S = min(4, n_ranges)
    ks = max(1, k // S) if floor else -(-k // S)
    thr = math.inf
    for y in range(S):
        r = y * n_ranges // S
        seg = scores[r * RANGE:(r + 1) * RANGE]
        pos = np.sort(seg[seg > 0])[::-1]
        if len(pos) >= ks:
            t = float((bits(pos[ks - 1:ks]) & np.uint64(~((1 << 40) - 1) & 0xFFFFFFFFFFFFFFFF)).view(np.float64)[0])
        else:
            t = 5e-324
        thr = min(thr, t)
    return thr


def candidates(scores, k, floor=False):
    return np.flatnonzero((scores > 0) & (scores >= sample_bound(scores, k, floor)))


def model_row(scores, k, defect=None):
    """(order, scores) of one query as the kernel's collect + final select produce it."""
    cand = candidates(scores, k, defect == "sample_floor")
    if defect == "stage_only" and len(cand) > STAGE:
        # the defect keeps 12288 of the candidates, whichever: both ends are modelled, and either must be detected
        lo, hi = cand[:STAGE], cand[-STAGE:]
        return [_select(scores, lo, k, None), _select(scores, hi, k, None)]
    return [_select(scores, cand, k, defect)]


def _select(scores, cand, k, defect):
    s = scores[cand]
    if defect == "ties_desc":
        pick = cand[np.lexsort((-cand, -s))][:k]
        return pick[np.lexsort((pick, -scores[pick]))]
    return cand[np.lexsort((cand, -s))][:k]


def model_topk(case, defect=None, rows=None):
    """Expected (ids, scores bits, counts) of the chosen rows; a list of alternatives when a defect has several."""
    idx, q = case.idx, case.queries
    rows = range(len(q)) if rows is None else rows
    blocked = max(len(t) for t in q) > case.block_hint
    sbq = sub_batch_size(idx.n_docs, len(q), blocked)
    outs = [[]]
    for b in rows:
        src = b % sbq if defect == "sub_batch_0" else b
        s = model_scores(idx, q[src], defect)
        alts = model_row(s, case.k, defect)
        outs = [o + [(a, s)] for o in outs for a in alts]
    base = 0 if defect == "no_id_base" else case.id_base
    res = []
    for o in outs:
        ids, sc, cnt = padded([a for a, _ in o], [s for _, s in o], case.k, base)
        res.append((ids, bits(sc), cnt))
    return res


# ----------------------------------------------------------------------------------------------------------- cases
@dataclass
class Case:
    name: str
    idx: object
    queries: list             # term-id arrays
    k: int
    id_base: int = 0
    rows: list | None = None  # rows a GPU test checks against FastBM25 (None = all)
    block_hint: int = 1883    # query length above which the kernel uses term blocks (upper bound, for sub_batch_size)
    notes: dict = field(default_factory=dict)


def edge_positions(n):
    p = {0, n - 1}
    for m in range(0, n + 2, SUB):
        p |= {m - 1, m, m + 1}
    return np.asarray(sorted(x for x in p if 0 <= x < n), np.int64)


@functools.lru_cache(maxsize=None)
def range_edge_case(n, variant):
    """Term 1 at docs 0, n-1 and every multiple of 512 (and so of 8192) +-1; term 2 sparse; term 3 in every third doc
    (a head term once n >= 4096); doc lengths 1..5 so every score differs."""
    rng = np.random.default_rng(n)
    e = edge_positions(n)
    r = np.unique(rng.integers(0, n, max(1, n // 50)))
    h = np.arange(0, n, 3)
    doc = np.concatenate([e, r, h])
    term = np.concatenate([np.full(len(e), 1), np.full(len(r), 2), np.full(len(h), 3)])
    tf = np.concatenate([1 + e % 3, np.ones(len(r), np.int64), 1 + h % 2])
    idx = index_from_triples(n, doc, term, tf, fill=1 + np.arange(n) % 5, variant=variant)
    raw = [[1], [1, 2], [3, 1], [2, 1, UNKNOWN, 3, 1]]
    return Case(f"range_edge_{n}_{variant}", idx, [idx.term_ids(t) for t in raw], k=1000)


@functools.lru_cache(maxsize=None)
def strip_case(variant, n=300_000, B=1000):
    """300 k two-token docs and B = 1000 queries: several sub-batches, CTAs walking runs of ranges.  Eight edge terms share
    the docs at every multiple of 512 +-1 (every strip, sub-range and range starts at a multiple of 512); query b holds
    edge term b % 8 and five random terms, so its top 300 holds every posting of its edge term."""
    rng = np.random.default_rng(7)
    e = edge_positions(n)
    rd = np.repeat(np.arange(n), 2)
    rt = rng.integers(0, 2000, 2 * n)
    doc = np.concatenate([e, rd])
    term = np.concatenate([10_000 + np.arange(len(e)) % 8, rt])
    tf = np.concatenate([2 + e % 3, np.ones(2 * n, np.int64)])
    idx = index_from_triples(n, doc, term, tf, fill=0, variant=variant)
    raw = [[10_000 + b % 8, *rng.integers(0, 2000, 5)] for b in range(B)]
    sbq = sub_batch_size(n, B)
    rows = sorted({r for b0 in range(0, B, sbq) for r in (b0, min(b0 + sbq, B) - 1)} | set(range(0, B, 37)))
    return Case(f"strips_{variant}", idx, [idx.term_ids(t) for t in raw], k=300, rows=rows)


@functools.lru_cache(maxsize=None)
def head_case(n, variant):
    """Term 1 with df = ceil(n/4) (df*4 == n when 4 | n), term 2 with df = (n-1)//4 (df*4 == n-1 when n % 4 == 1), term 3
    in half the docs, term 4 a short list; queries: every order of (head, list, unknown, duplicate head)."""
    import itertools

    rng = np.random.default_rng(n + 1)
    parts = [(1, -(-n // 4)), (2, (n - 1) // 4), (3, n // 2), (4, max(1, n // 40))]
    doc, term, tf = [], [], []
    for t, df in parts:
        d = np.sort(rng.choice(n, df, replace=False))
        doc.append(d)
        term.append(np.full(df, t))
        tf.append(1 + d % 3)
    idx = index_from_triples(n, np.concatenate(doc), np.concatenate(term), np.concatenate(tf),
                             fill=1 + np.arange(n) % 4, variant=variant)
    raw = [list(p) for p in itertools.permutations([3, 4, UNKNOWN, 3])]
    raw = [r + [1, 2] if i % 2 else [2] + r + [1] for i, r in enumerate(raw)]
    return Case(f"head_{n}_{variant}", idx, [idx.term_ids(t) for t in raw], k=100)


@functools.lru_cache(maxsize=None)
def many_heads_case(variant, n=8192, n_heads=70):
    """70 head terms with distinct df (the 6 smallest get no dense row), interleaved with list and unknown terms."""
    rng = np.random.default_rng(70)
    doc, term = [], []
    for j in range(n_heads):
        d = rng.choice(n, n // 4 + 8 * j, replace=False)
        doc.append(d)
        term.append(np.full(len(d), 100 + j))
    lst = rng.choice(n, 300, replace=False)
    doc = np.concatenate(doc + [lst])
    term = np.concatenate(term + [np.full(300, 5)])
    idx = index_from_triples(n, doc, term, 1 + doc % 2, fill=1 + np.arange(n) % 3, variant=variant)
    raw = [[100, 5, 169, UNKNOWN, 101, 100, 164, 102], [103, 104, 105], [168, 100 + 63, 100 + 64, 5, 5],
           list(range(100, 170)), [5, UNKNOWN, 102, 169, 101]]
    return Case(f"many_heads_{variant}", idx, [idx.term_ids(t) for t in raw], k=200)


LONG_LENGTHS = (1, 511, 512, 513, 1025, 1871, 1872, 1883, 1884, 5000, 20000)


@functools.lru_cache(maxsize=None)
def long_query_case(variant, n=20_000):
    """Queries of 1 .. 20000 terms in one batch (random known terms, duplicates and unknown tokens)."""
    rng = np.random.default_rng(11)
    dl = rng.integers(3, 12, n)
    d = np.repeat(np.arange(n), dl)
    t = (rng.zipf(1.3, len(d)) - 1) % 6000
    idx = index_from_triples(n, d, t, 1, fill=0, variant=variant)
    raw = [rng.integers(0, 6500, L) for L in LONG_LENGTHS]   # ids >= 6000 are unknown
    return Case(f"long_{variant}", idx, [idx.term_ids(r) for r in raw], k=100)


@functools.lru_cache(maxsize=None)
def k_sweep_case(variant, k, n=3 * RANGE + 1):
    rng = np.random.default_rng(k)
    d = np.repeat(np.arange(n), 3)
    t = rng.integers(0, 3000, len(d))
    rare = np.array([5, 900, 4000, n - 1])
    idx = index_from_triples(n, np.concatenate([d, rare]), np.concatenate([t, np.full(4, 9999)]), 1, fill=0,
                             variant=variant)
    raw = [list(rng.integers(0, 3000, 6)) for _ in range(6)] + [[9999], [9999, UNKNOWN]]
    return Case(f"k{k}_{variant}", idx, [idx.term_ids(r) for r in raw], k=k)


@functools.lru_cache(maxsize=None)
def tie_case(m, variant, n=100_000):
    """Equal doc lengths, one term with tf = 1 in m docs spread over the corpus: m exactly tied candidates."""
    d = np.unique(np.linspace(0, n - 1, m).astype(np.int64))
    assert len(d) == m
    idx = index_from_triples(n, d, np.full(m, 1), 1, fill=(~np.isin(np.arange(n), d)).astype(np.int64),
                             variant=variant)
    return Case(f"ties_{m}_{variant}", idx, [idx.term_ids([1]), idx.term_ids([1, UNKNOWN])], k=1000)


@functools.lru_cache(maxsize=None)
def both_ends_case(variant, n=100_000, m=40_000):
    """40000 tied docs and 20 better docs at both ends of the corpus (docs 0..9 and n-10..n-1 hold the term twice)."""
    d = np.unique(np.linspace(0, n - 1, m).astype(np.int64))
    ends = np.concatenate([np.arange(10), np.arange(n - 10, n)])
    d = np.unique(np.concatenate([d, ends]))
    tf = np.where(np.isin(d, ends), 2, 1)
    fill = (~np.isin(np.arange(n), d)).astype(np.int64)
    idx = index_from_triples(n, d, np.full(len(d), 1), tf, fill=fill, variant=variant)
    return Case(f"both_ends_{variant}", idx, [idx.term_ids([1])], k=1000)


@functools.lru_cache(maxsize=None)
def straddle_case(variant, n=5 * RANGE - 1):
    """300 docs with tf 2 and a 500-doc tie group spread over all five ranges: rank k = 500 falls inside the ties.
    Ids are reported from id_base = 2^40."""
    rng = np.random.default_rng(5)
    d = np.sort(rng.choice(n, 800, replace=False))
    tf = np.where(np.arange(800) % 8 < 3, 2, 1)
    idx = index_from_triples(n, d, np.full(800, 1), tf, fill=np.where(np.isin(np.arange(n), d), 0, 1),
                             variant=variant)
    return Case(f"straddle_{variant}", idx, [idx.term_ids([1]), idx.term_ids([1, 1])], k=500, id_base=1 << 40)


@functools.lru_cache(maxsize=None)
def sample_case(kind):
    """Okapi only (BM25Plus makes every doc positive).
    * ``empty_sampled``: five ranges, positives only in range 4, which is not sampled (samples: ranges 0, 1, 2, 3).
    * ``exact_ks``: the sampled ranges hold exactly ceil(k/S) = 3 low-scoring positives each, the top k lies in range 4.
    * ``tight``: four ranges, each with 2 high docs and 1 low doc: the bound is the low score, exactly tight at k = 10."""
    n = 5 * RANGE if kind != "tight" else 4 * RANGE
    rng = np.random.default_rng(len(kind))
    hi_docs, lo_docs = [], []
    if kind == "empty_sampled":
        hi_docs = 4 * RANGE + np.sort(rng.choice(RANGE, 50, replace=False))
    elif kind == "exact_ks":
        hi_docs = 4 * RANGE + np.sort(rng.choice(RANGE, 20, replace=False))
        lo_docs = np.concatenate([r * RANGE + np.sort(rng.choice(RANGE, 3, replace=False)) for r in range(4)])
    else:
        for r in range(4):
            c = r * RANGE + np.sort(rng.choice(RANGE, 3, replace=False))
            hi_docs += list(c[:2])
            lo_docs += [c[2]]
    hi_docs, lo_docs = np.asarray(hi_docs, np.int64), np.asarray(lo_docs, np.int64)
    fill = np.ones(n, np.int64)
    fill[lo_docs] = 8          # long docs: a low BM25 ratio
    idx = index_from_triples(n, np.concatenate([hi_docs, lo_docs]),
                             np.concatenate([np.full(len(hi_docs), 1), np.full(len(lo_docs), 2)]), 1, fill=fill)
    raw = [[1, 2, 1, 1], [2], [1]]
    return Case(f"sample_{kind}", idx, [idx.term_ids(r) for r in raw], k=10)


@functools.lru_cache(maxsize=None)
def extreme_case(kind, variant="okapi"):
    rng = np.random.default_rng(3)
    kw = {}
    if kind == "idf_zero":            # Okapi: N = 2 df  ->  log(N - df + 0.5) - log(df + 0.5) == 0.0 exactly
        n = 40
        doc = np.concatenate([np.arange(0, n, 2), [1, 3, 5]])
        term = np.concatenate([np.full(n // 2, 1), [2, 2, 2]])
        tf = 1
    elif kind == "negative_floor":    # average idf < 0: the epsilon floor is negative
        n = 10
        doc = np.concatenate([np.arange(9), np.arange(1, 9), [4]])
        term = np.concatenate([np.full(9, 1), np.full(8, 2), [3]])
        tf = np.concatenate([np.ones(17, np.int64), [1]])
        idx = index_from_triples(n, doc, term, tf, fill=0, variant=variant)
        return Case(f"negative_floor_{variant}", idx, [idx.term_ids(r) for r in ([1], [1, 2], [2, 1, 1], [3], [1, 3])],
                    k=10)
    elif kind == "empty_docs":
        n = 9000
        live = np.flatnonzero(rng.random(n) < 0.6)
        doc = np.repeat(live, 2)
        term = rng.integers(0, 40, len(doc))
        tf = 1
        fill = np.zeros(n, np.int64)
        idx = index_from_triples(n, doc, term, tf, fill=fill, variant=variant)
        return Case(f"empty_docs_{variant}", idx, [idx.term_ids(list(rng.integers(0, 40, 4))) for _ in range(5)], k=1024)
    elif kind == "tf_max":
        n = 5000
        rest = np.arange(3, n - 2, 7)
        doc = np.concatenate([[0, n - 1, 2500], rest])
        term = np.concatenate([[1, 1, 2], np.full(len(rest), 1)])
        tf = np.concatenate([[65535, 65535, 65535], np.ones(len(rest), np.int64)])
    else:                             # (k1, b) parameter edges
        k1, b = {"k1_0": (0.0, 0.75), "b_0": (1.5, 0.0), "b_1": (1.5, 1.0)}[kind]
        kw = dict(k1=k1, b=b)
        n = 20000
        doc = np.repeat(np.arange(n), 2)
        term = rng.integers(0, 500, len(doc))
        tf = 1
    idx = index_from_triples(n, doc, term, tf, fill=1 + np.arange(n) % 3, variant=variant, **kw)
    raw = [[1], [1, 2], [2, 1, 2], list(range(10)), [UNKNOWN]]
    return Case(f"{kind}_{variant}", idx, [idx.term_ids(r) for r in raw], k=64)
