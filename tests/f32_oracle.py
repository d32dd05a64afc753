"""Exact fp64 top-k on float32 storage (TEST INFRASTRUCTURE, DESIGN.md K1g).

Restates what Qdrant returns for a collection whose ``VectorParams.datatype`` is float32 (its default): every score is
evaluated on the vectors as given, x, and the fp32 query q, in fp64:
    Cosine  <q, x> / (||q|| ||x||)   (0 for a zero row or a zero query), best first
    Dot     <q, x>                    best first
    Euclid  ||q - x||                 nearest first, computed directly
Ties by ascending row.  No fp16 rounding enters anywhere.
"""
from __future__ import annotations

import numpy as np


def f32_scores(x: np.ndarray, q: np.ndarray, metric: str) -> np.ndarray:
    x64 = np.asarray(x, dtype=np.float32).astype(np.float64)
    q64 = np.asarray(q, dtype=np.float32).astype(np.float64)
    if metric == "euclid":
        out = np.empty(len(x64))
        for r0 in range(0, len(x64), 4096):   # direct differences, chunked to bound memory
            t = q64[None, :] - x64[r0:r0 + 4096]
            out[r0:r0 + 4096] = np.sqrt((t * t).sum(axis=1))
        return out
    dot = x64 @ q64
    if metric == "dot":
        return dot
    den = np.sqrt((x64 * x64).sum(axis=1)) * np.sqrt(q64 @ q64)
    out = np.zeros(len(x64))
    np.divide(dot, den, out=out, where=den > 0.0)
    return out


def f32_topk(x, q, k, metric, rows=None):
    """(row indices, scores) of the exact top-k; ``rows`` restricts the candidates (a filter's matching rows)."""
    return f32_topk_many(x, np.asarray(q)[None, :], k, metric, rows=rows)[0]


def f32_topk_many(x, qs, k, metric, rows=None):
    """``f32_topk`` of every query in ``qs``, with the corpus widened to fp64 once: [(rows, scores) per query].
    Euclid keeps only the rows whose fp64 expansion ||x||^2 - 2 <q, x> is within 2 m of the k-th smallest, m a generous
    bound on the expansion's error, and scores those directly: every excluded row is strictly farther than the k-th
    (exact ties, such as every row of a query of norm 1e30, keep all their rows)."""
    idx = np.arange(len(x)) if rows is None else np.asarray(rows, dtype=np.int64)
    x64 = np.asarray(x, dtype=np.float32)[idx].astype(np.float64)
    q64 = np.asarray(qs, dtype=np.float32).astype(np.float64)
    gram = x64 @ q64.T
    xx = (x64 * x64).sum(axis=1)
    out = []
    for b in range(len(q64)):
        qq = float(q64[b] @ q64[b])
        if metric == "euclid":
            cand = np.arange(len(idx))
            if len(idx) > k:
                a = xx - 2.0 * gram[:, b]
                m = 1e-12 * (qq + float(xx.max()))
                cand = np.flatnonzero(a <= np.partition(a, k - 1)[k - 1] + 2.0 * m)
            t = q64[b][None, :] - x64[cand]
            s = np.sqrt((t * t).sum(axis=1))
            key = s
        else:
            cand = np.arange(len(idx))
            s = gram[:, b].copy()
            if metric == "cosine":
                den = np.sqrt(xx) * np.sqrt(qq)
                s = np.zeros(len(idx))
                np.divide(gram[:, b], den, out=s, where=den > 0.0)
            key = -s
        o = np.lexsort((idx[cand], key))[:k]
        out.append((idx[cand][o], s[o]))
    return out


def f32_max_norm(x):
    return float(np.sqrt((np.asarray(x, np.float64) ** 2).sum(axis=1)).max()) if len(x) else 0.0


def f32_magnitude(xmax, q, metric):
    """The size of the terms a score is computed from (the absolute tolerance of ``assert_metric_topk`` scales with
    it): 1 (cosine), ||q|| xmax (dot), ||q|| + xmax (euclid); xmax = ``f32_max_norm`` of the rows."""
    if metric == "cosine":
        return 1.0
    qn = float(np.linalg.norm(np.asarray(q, np.float64)))
    return qn * xmax if metric == "dot" else qn + xmax
