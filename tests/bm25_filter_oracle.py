"""Reference of filtered BM25 (``sb_bm25_topk_filtered``, DESIGN.md K2 "Filtered BM25 and hybrid") for its tests
(TEST INFRASTRUCTURE).

* ``csr``           -- per-query lists of (field, code) conditions -> the (f_off, f_field, f_code) int32 CSR of the C ABI.
* ``match_mask``    -- the docs that satisfy one query's conditions: tags[field][doc] == code >= 0 for every condition
                       (no condition: every doc).
* ``filtered_topk`` -- the unfiltered rank_bm25 order (stable ``argsort(-s)``, ties by ascending doc, ``s > 0``)
                       restricted to the matching docs, first k.
* ``padded``        -- rows in the kernel's output layout (ids + id_base / -1, scores / 0.0, counts).
"""
from __future__ import annotations

import numpy as np


def csr(cond_lists):
    off = np.zeros(len(cond_lists) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in cond_lists])
    fld = np.asarray([f for c in cond_lists for f, _ in c], np.int32)
    code = np.asarray([v for c in cond_lists for _, v in c], np.int32)
    return off, fld, code


def match_mask(tags, conds, n):
    m = np.ones(n, bool)
    for f, c in conds:
        m &= (tags[f] == c) if c >= 0 else np.zeros(n, bool)
    return m


def filtered_topk(scores, match, k):
    order = np.argsort(-scores, kind="stable")
    return order[match[order] & (scores[order] > 0)][:k]


def padded(orders, scores_list, k, id_base=0):
    B = len(orders)
    ids = np.full((B, k), -1, np.int64)
    sc = np.zeros((B, k))
    cnt = np.zeros(B, np.int32)
    for b, (o, s) in enumerate(zip(orders, scores_list)):
        ids[b, :len(o)] = o + id_base
        sc[b, :len(o)] = s[o]
        cnt[b] = len(o)
    return ids, sc, cnt
