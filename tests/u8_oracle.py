"""Exact fp64 top-k on uint8 storage (TEST INFRASTRUCTURE, DESIGN.md K1i).

Restates what a collection whose ``VectorParams.datatype`` is uint8 returns: every score is evaluated in fp64 on the
stored integer vector x (components in [0, 255]) and the fp32 query q as given:
    Cosine  <q, x> / (||q|| ||x||)   (0 for a zero row or a zero query), best first
    Dot     <q, x>                    best first
    Euclid  ||q - x||                 nearest first, computed directly
Ties by ascending row.  These are the float32-storage formulas on x widened exactly, so the float32 oracle computes
them; ``u8_brute_topk`` is a second, independent statement used to check it.
"""
from __future__ import annotations

import numpy as np

from f32_oracle import f32_magnitude, f32_max_norm, f32_scores, f32_topk, f32_topk_many  # noqa: F401


def _x(x):
    x = np.asarray(x)
    assert x.dtype == np.uint8, "a uint8 corpus"
    return x.astype(np.float32)


def u8_scores(x, q, metric):
    return f32_scores(_x(x), q, metric)


def u8_topk(x, q, k, metric, rows=None):
    return f32_topk(_x(x), q, k, metric, rows=rows)


def u8_topk_many(x, qs, k, metric, rows=None):
    return f32_topk_many(_x(x), qs, k, metric, rows=rows)


def u8_magnitude(x, q, metric):
    return f32_magnitude(f32_max_norm(_x(x)), q, metric)


def u8_brute_topk(x, q, k, metric):
    """Row by row in Python floats (fp64), sorted by (key, row): slow, for small corpora only."""
    qv = [float(v) for v in np.asarray(q, np.float32)]
    qn = sum(v * v for v in qv) ** 0.5
    out = []
    for r, row in enumerate(np.asarray(x, np.uint8).tolist()):
        if metric == "euclid":
            s = sum((a - b) ** 2 for a, b in zip(qv, row)) ** 0.5
            out.append((s, r, s))
            continue
        dot = sum(a * b for a, b in zip(qv, row))
        if metric == "dot":
            s = dot
        else:
            den = qn * sum(b * b for b in row) ** 0.5
            s = dot / den if den > 0 else 0.0
        out.append((-s, r, s))
    out.sort()
    return np.asarray([r for _, r, _ in out[:k]], np.int64), np.asarray([s for _, _, s in out[:k]])


def clustered_corpus(n, d, seed, centers=64):
    """Quantised nonnegative rows round(128 + 40 g), clipped to [0, 255], g Gaussian around a few centres: cosines
    sit in a narrow band."""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centers, d))
    g = c[rng.integers(0, centers, n)] * 0.5 + rng.standard_normal((n, d))
    return np.clip(np.rint(128 + 40 * g), 0, 255).astype(np.uint8)


def u8_query_column(c):
    """Mirror of the kernel's column permutation (dense_common.cuh): natural column c of a 64-column block -> its
    column in the permuted fp16 query block."""
    t, s, j = c >> 4, (c >> 2) & 3, c & 3
    return 16 * s + 2 * t + (j if j < 2 else 6 + j)
