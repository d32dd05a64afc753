"""Exact fp64 Dot / Euclid top-k over the stored representation (TEST INFRASTRUCTURE, DESIGN.md K1e).

Restates what the reference obtains from Qdrant for a collection created with distance="Dot" or "Euclid"
(src/core/vector_store/qdrant_store.py:52, 224-237), evaluated exactly in fp64 on the vector the store keeps:
    y = fp16(x / ||x||)        (the Cosine row, fp64 normalisation, one rounding; fp16 input is normalised too)
    c = ||x|| / ||y||          (fp64; 0 for a zero row)
    v = c * y
Dot scores <q, v> (q as given), best first; Euclid scores ||q - v||, nearest first; ties by ascending row.
"""
from __future__ import annotations

import numpy as np


def stored_metric(vecs: np.ndarray):
    """(y [n, d] fp16, c [n] fp64) the store keeps for these input rows under Dot / Euclid."""
    x = np.asarray(vecs)
    x64 = x.astype(np.float64) if x.dtype == np.float16 else x.astype(np.float32).astype(np.float64)
    nrm = np.sqrt((x64 * x64).sum(axis=1))
    safe = np.where(nrm > 0.0, nrm, 1.0)
    y = (x64 / safe[:, None]).astype(np.float16)
    y64 = y.astype(np.float64)
    yn = np.sqrt((y64 * y64).sum(axis=1))
    c = np.zeros(len(x64))
    np.divide(nrm, yn, out=c, where=yn > 0.0)
    return y, c


def metric_scores(y: np.ndarray, c: np.ndarray, q: np.ndarray, metric: str) -> np.ndarray:
    """fp64 score of every stored row: <q, v> (dot) or ||q - v|| (euclid)."""
    q64 = np.asarray(q, dtype=np.float32).astype(np.float64)
    y64 = y.astype(np.float64)
    if metric == "dot":
        return c * (y64 @ q64)
    diff = q64[None, :] - c[:, None] * y64
    return np.sqrt((diff * diff).sum(axis=1))


def metric_topk(y, c, q, k, metric, rows=None):
    """(row indices, scores) of the exact top-k; ``rows`` restricts the candidates (a filter's matching rows)."""
    s = metric_scores(y, c, q, metric)
    idx = np.arange(len(s)) if rows is None else np.asarray(rows, dtype=np.int64)
    key = -s[idx] if metric == "dot" else s[idx]
    o = np.lexsort((idx, key))[:k]
    return idx[o], s[idx[o]]


def magnitude(c, q, rows, metric):
    """The size of the terms a score is computed from: ||q|| max ||v|| (dot) or ||q|| + max ||v|| (euclid, whose
    distance of a query close to a row cancels down to far below either norm)."""
    qn = float(np.linalg.norm(np.asarray(q, np.float64)))
    vmax = float(np.max(c[rows])) * (1.0 + 2.0 ** -10) if len(rows) else 0.0
    return qn * vmax if metric == "dot" else qn + vmax


def assert_metric_topk(ids, scores, count, want_ids, want_scores, what="", rtol=1e-9, tie_rel=1e-12, mag=None):
    """Ids equal and scores within rtol, with the absolute tolerance scaled to the score magnitude (``mag``, default
    the largest score; see ``magnitude``); inside a group of oracle scores tied to fp64 precision any order is accepted.
    The device and the oracle sum ||x|| in different orders, so their c (and v) may differ in the last bit."""
    n = int(count)
    assert n == len(want_ids), f"{what}: count {n} != {len(want_ids)}"
    got_sc = np.asarray(scores[:n], dtype=np.float64)
    want_sc = np.asarray(want_scores, dtype=np.float64)
    scale = max(1e-300, float(np.abs(want_sc).max())) if n else 1.0
    if mag is not None:
        scale = max(scale, mag)
    assert np.allclose(got_sc, want_sc, rtol=rtol, atol=1e-12 * scale), \
        f"{what}: scores differ, max |diff| {np.abs(got_sc - want_sc).max() if n else 0}"
    got_ids = list(map(int, ids[:n]))
    if got_ids == list(map(int, want_ids)):
        return
    i = 0
    while i < n:
        j = i
        while j + 1 < n and abs(want_sc[j + 1] - want_sc[i]) <= tie_rel * scale:
            j += 1
        assert sorted(got_ids[i:j + 1]) == sorted(map(int, want_ids[i:j + 1])), \
            f"{what}: rank {i}..{j}: {got_ids[i:j + 1]} vs {list(want_ids[i:j + 1])}"
        i = j + 1
