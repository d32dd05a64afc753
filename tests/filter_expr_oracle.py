"""The semantics of ``query_points`` filters, restated twice for the tests:

* ``matches(flt, payload)`` evaluates a filter on one payload dict, row by row, straight from the filter objects
  (Python comparisons, typed equality) -- the contract of INTEGRATION.md's semantics table;
* ``run_programs(p_off, prog, pool, tags, vals, n)`` interprets compiled predicate programs (``sb_pred``) over tag and
  value columns in NumPy -- what the mask kernel must compute.

Neither imports the product's compiler, so a test that compares them checks ``PayloadIndex.compile_programs``.
"""
from __future__ import annotations

import math

import numpy as np

EQ, IN, RANGE, PRESENT, AND, OR, NOR, ATLEAST = 1, 2, 3, 4, 5, 6, 7, 8
_MISSING = object()


def value_at(payload, key):
    cur = payload
    for part in key.split("."):
        if not isinstance(cur, dict) or part not in cur:
            return _MISSING
        cur = cur[part]
    return cur


def _is_filter(x):
    return any(hasattr(x, a) for a in ("must", "should", "must_not", "min_should"))


def _list(x):
    if x is None:
        return []
    return list(x) if isinstance(x, (list, tuple)) else [x]


def _typed_eq(v, x):
    return type(v) is type(x) and v == x


def _numeric(v):
    return isinstance(v, (int, float)) and not isinstance(v, bool) and not (isinstance(v, float) and math.isnan(v))


def _condition(c, payload):
    if _is_filter(c):
        return matches(c, payload)
    v = value_at(payload, c.key)
    r = getattr(c, "range", None)
    if r is not None:
        if not _numeric(v):
            return False
        return all(ok for ok in ((r.gt is None or v > r.gt), (r.gte is None or v >= r.gte),
                                 (r.lt is None or v < r.lt), (r.lte is None or v <= r.lte)))
    m = c.match
    if v is _MISSING or v is None:
        return False
    if getattr(m, "any", None) is not None:
        return any(_typed_eq(v, x) for x in m.any)
    return _typed_eq(v, m.value)


def matches(flt, payload) -> bool:
    """True iff the payload satisfies the filter (None: every payload)."""
    if flt is None:
        return True
    if not _is_filter(flt):
        return _condition(flt, payload)
    if not all(_condition(c, payload) for c in _list(getattr(flt, "must", None))):
        return False
    should = _list(getattr(flt, "should", None))
    if should and not any(_condition(c, payload) for c in should):
        return False
    if any(_condition(c, payload) for c in _list(getattr(flt, "must_not", None))):
        return False
    ms = getattr(flt, "min_should", None)
    if ms is not None and sum(_condition(c, payload) for c in _list(ms.conditions)) < ms.min_count:
        return False
    return True


def run_programs(p_off, prog, pool, tags: dict, vals: dict, n: int) -> np.ndarray:
    """bool [B, n]: row r of query b matches iff program prog[p_off[b]:p_off[b+1]] leaves a 1 (empty: every row).
    ``tags[f]`` int32 [n] (code, -1 = absent), ``vals[f]`` float64 [n] (NaN = no value)."""
    B = len(p_off) - 1
    out = np.ones((B, n), bool)
    for b in range(B):
        stack = []
        for e in prog[p_off[b]:p_off[b + 1]]:
            op = int(e["op"])
            if op == EQ:
                stack.append(tags[int(e["field"])] == int(e["a"]))
            elif op == IN:
                codes = pool[int(e["a"]):int(e["a"]) + int(e["b"])]
                assert np.all(np.diff(codes) > 0) and np.all(codes >= 0)
                stack.append(np.isin(tags[int(e["field"])], codes))
            elif op == PRESENT:
                stack.append(tags[int(e["field"])] >= 0)
            elif op == RANGE:
                v = vals[int(e["field"])]
                with np.errstate(invalid="ignore"):
                    lo = v >= e["lo"] if e["lo_incl"] else v > e["lo"]
                    hi = v <= e["hi"] if e["hi_incl"] else v < e["hi"]
                stack.append(lo & hi)
            else:
                na = int(e["a"])
                args = stack[len(stack) - na:] if na else []
                del stack[len(stack) - na:]
                s = np.sum(args, axis=0) if na else np.zeros(n, np.int64)
                stack.append({AND: s == na, OR: s > 0, NOR: s == 0, ATLEAST: s >= int(e["b"])}[op])
            assert len(stack) <= 64
        if p_off[b + 1] > p_off[b]:
            assert len(stack) == 1
            out[b] = stack[0]
    return out
