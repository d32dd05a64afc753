"""Exact grouped search, written as its definition (TEST INFRASTRUCTURE, DESIGN.md K1f).

Qdrant's ``search_groups(group_by=, limit=L, group_size=G)``: sort every matching row exactly (score descending, or
distance ascending for Euclid; ties by ascending row), walk the list, and keep each row whose group is among the first L
distinct groups seen and which is among its group's first G rows.  A row in no group (None) is skipped.
"""
from __future__ import annotations

import numpy as np


def group_search(scores, groups, limit, group_size, rows=None, ascending=False):
    """[(group, [(row, score), ...]), ...] best group first.  ``scores``: fp64 per row; ``groups``: one hashable group
    per row, None = no group; ``rows``: the candidate rows (a filter's matches), default all."""
    s = np.asarray(scores, dtype=np.float64)
    idx = np.arange(len(s)) if rows is None else np.asarray(rows, dtype=np.int64)
    order = idx[np.lexsort((idx, s[idx] if ascending else -s[idx]))]
    hits: dict = {}
    seen: list = []
    for r in order.tolist():
        g = groups[r]
        if g is None:
            continue
        if g not in hits:
            if len(seen) == limit:
                continue
            hits[g] = []
            seen.append(g)
        if len(hits[g]) < group_size:
            hits[g].append((r, float(s[r])))
    return [(g, hits[g]) for g in seen]
