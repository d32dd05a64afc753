"""Exact fp64 recommendation oracle (TEST INFRASTRUCTURE, DESIGN.md K1j).

Similarities are evaluated on the rows as the slot stores them: a float16 slot's fp16 row y (Cosine) or c * y (Dot,
tests/metric_oracle.py), a float32 slot's x, a uint8 slot's integers.  The merge follows INTEGRATION.md:
    best_score: p = max over positives, n = max over negatives (-inf when empty); g(p) if p > n else -g(n),
                g(x) = 0.5 (x / (1 + |x|) + 1)
    sum_scores: (sum over positives, in order) - (sum over negatives, in order)
Order: score descending, row ascending.
"""
from __future__ import annotations

import math

import numpy as np

from metric_oracle import stored_metric


def g(x: float) -> float:
    return 0.5 * (x / (1.0 + abs(x)) + 1.0)


def best(p: float, n: float) -> float:
    return g(p) if p > n else -g(n)


def stored(x, storage: str, metric: str):
    """(rows fp64 [n, d], per-row factor) so that the similarity of query q is factor * (rows @ q) (Dot) or the
    cosine of q and rows (Cosine)."""
    if storage == "float16":
        y, c = stored_metric(x)
        y64 = y.astype(np.float64)
        return y64, (c if metric == "dot" else None)
    return np.asarray(x).astype(np.float64), None


def similarities(rows, fac, e, metric: str) -> np.ndarray:
    q = np.asarray(e, np.float32).astype(np.float64)
    dot = rows @ q
    if metric == "dot":
        return dot if fac is None else fac * dot
    den = np.sqrt((rows * rows).sum(1)) * math.sqrt(float(q @ q))
    return np.divide(dot, den, out=np.zeros_like(dot), where=den > 0)


def merged(S: np.ndarray, n_pos: int, strategy: str) -> np.ndarray:
    """S [n, m] similarities -> merged scores [n], the terms taken in example order."""
    n, m = S.shape
    if strategy == "sum_scores":
        sp, sn = np.zeros(n), np.zeros(n)
        for j in range(m):
            if j < n_pos:
                sp = sp + S[:, j]
            else:
                sn = sn + S[:, j]
        return sp - sn
    p = S[:, :n_pos].max(1) if n_pos else np.full(n, -np.inf)
    q = S[:, n_pos:].max(1) if n_pos < m else np.full(n, -np.inf)
    with np.errstate(invalid="ignore"):   # the branch not taken may be g(-inf)
        return np.where(p > q, 0.5 * (p / (1 + np.abs(p)) + 1), -0.5 * (q / (1 + np.abs(q)) + 1))


def reco_topk(rows, fac, examples, n_pos, strategy, metric, k, cand=None):
    """(rows, scores) of the exact top-k; ``cand`` restricts the candidates (a filter's matching rows)."""
    S = np.stack([similarities(rows, fac, e, metric) for e in examples], 1)
    s = merged(S, n_pos, strategy)
    idx = np.arange(len(s)) if cand is None else np.asarray(cand, np.int64)
    o = np.lexsort((idx, -s[idx]))[:k]
    return idx[o], s[idx[o]]


def reco_brute(rows, fac, examples, n_pos, strategy, metric, k):
    """Independent row-by-row restatement with Python floats (small corpora only)."""
    out = []
    for i, r in enumerate(rows):
        sims = []
        for e in examples:
            q = [float(v) for v in np.asarray(e, np.float32)]
            dot = math.fsum(a * b for a, b in zip(r.tolist(), q))
            if metric == "dot":
                sims.append(dot * (1.0 if fac is None else float(fac[i])))
            else:
                den = math.sqrt(math.fsum(a * a for a in r.tolist())) * math.sqrt(math.fsum(b * b for b in q))
                sims.append(dot / den if den > 0 else 0.0)
        if strategy == "sum_scores":
            sc = math.fsum(sims[:n_pos]) - math.fsum(sims[n_pos:])
        else:
            sc = best(max(sims[:n_pos], default=-math.inf), max(sims[n_pos:], default=-math.inf))
        out.append((-sc, i))
    out.sort()
    return np.array([i for _, i in out[:k]], np.int64), np.array([-s for s, _ in out[:k]])
