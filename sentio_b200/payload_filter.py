"""Payload filters of the Qdrant search API, compiled for the filtered dense scan (``sb_dense_topk_filtered``), and the
boolean filters of ``query_points``, compiled into predicate programs (``sb_dense_topk_where``, DESIGN.md K1h).

The reference filters its searches with ``client.search(..., query_filter=_convert_filter(filter))``
(src/core/vector_store/qdrant_store.py:120-146, 351-381); ``_convert_filter`` (:456-471) turns ``{"source": "a.pdf"}``
into ``FieldCondition(key="metadata.source", match=MatchValue(value="a.pdf"))`` and several keys into
``Filter(must=[...])``.  That is the supported subset: a conjunction of "payload key == scalar value" conditions.
Everything else (``should``, ``must_not``, ranges, ``MatchAny``, nested filters, list-valued payload fields, non-scalar
values) raises ``ValueError`` naming the unsupported part -- it is never ignored.

``compile_programs`` (``query_points``) reads the richer language: ``must`` / ``should`` / ``must_not`` / ``min_should``,
nested filters, ``MatchValue``, ``MatchAny`` and ``Range`` (semantics in INTEGRATION.md; ``tests/filter_expr_oracle.py``
restates them row by row).  Its leaves read tag columns (dictionary codes) and numeric value columns (fp64, NaN = no
value), both built lazily per key.

``qdrant_client`` is not a dependency: filters are read by duck typing (``.must``, ``.key``, ``.match.value``), so the
real Qdrant models and any object of the same shape work.
"""
from __future__ import annotations

from typing import Any, Sequence

import numpy as np

MAX_TAG_FIELDS = 16     # SB_MAX_TAG_FIELDS (include/sentio_b200.h)
MAX_VALUE_FIELDS = 16   # SB_MAX_VALUE_FIELDS
MAX_CONDITIONS = 64     # conditions per filter, nested filters and their conditions included
MAX_DEPTH = 8           # nesting depth of filters (a filter without nested filters has depth 1)
MAX_ANY = 1024          # values per MatchAny
MAX_STACK = 64          # SB_MAX_PRED_STACK
EXACT_INT = 2 ** 53     # ints up to this magnitude are exact in fp64

# one program step: struct sb_pred of include/sentio_b200.h
PRED_DTYPE = np.dtype([("op", "<i4"), ("field", "<i4"), ("a", "<i4"), ("b", "<i4"), ("lo", "<f8"), ("hi", "<f8"),
                       ("lo_incl", "<i4"), ("hi_incl", "<i4")])
EQ, IN, RANGE, PRESENT, AND, OR, NOR, ATLEAST = 1, 2, 3, 4, 5, 6, 7, 8   # SB_PRED_*
_MISSING = object()


def value_key(v: Any):
    """Dictionary key of a payload value: typed, so ``True`` and ``1`` (equal in Python) get different codes."""
    return (type(v).__name__, v)


def _check_value(v: Any, key: str):
    if isinstance(v, bool):
        return bool(v)
    if isinstance(v, int):
        return int(v)
    if isinstance(v, str):
        return str(v)
    raise ValueError(f"query_filter: condition on {key!r} has a non-scalar value of type {type(v).__name__} "
                     "(only str, int and bool are supported)")


def _empty(x) -> bool:
    return x is None or (isinstance(x, (list, tuple)) and len(x) == 0)


def _condition(c, where: str):
    if hasattr(c, "must") or hasattr(c, "should") or hasattr(c, "must_not"):
        raise ValueError(f"query_filter: nested Filter in {where} is not supported")
    key = getattr(c, "key", None)
    if not isinstance(key, str) or not key:
        raise ValueError(f"query_filter: {where} entry {type(c).__name__} is not a FieldCondition with a key")
    for attr in ("range", "geo_bounding_box", "geo_radius", "geo_polygon", "values_count", "datetime_range"):
        if getattr(c, attr, None) is not None:
            raise ValueError(f"query_filter: condition on {key!r} uses {attr}, which is not supported")
    m = getattr(c, "match", None)
    if m is None:
        raise ValueError(f"query_filter: condition on {key!r} has no match (only MatchValue is supported)")
    for attr in ("any", "except_", "text", "phrase"):
        if getattr(m, attr, None) is not None:
            raise ValueError(f"query_filter: condition on {key!r} uses {type(m).__name__}.{attr} "
                             "(only MatchValue is supported)")
    if not hasattr(m, "value"):
        raise ValueError(f"query_filter: condition on {key!r} uses {type(m).__name__} (only MatchValue is supported)")
    return key, _check_value(m.value, key)


def compile_filter(flt) -> list[tuple[str, Any]]:
    """``Filter(must=[FieldCondition...])`` or a bare ``FieldCondition`` -> [(key, value), ...]; ``None`` -> []."""
    if flt is None:
        return []
    if not hasattr(flt, "must") and hasattr(flt, "key"):   # _convert_filter returns a bare condition for one key
        return [_condition(flt, "query_filter")]
    if not (hasattr(flt, "must") or hasattr(flt, "should") or hasattr(flt, "must_not")):
        raise ValueError(f"query_filter: unsupported filter object of type {type(flt).__name__}")
    for attr in ("should", "must_not", "min_should"):
        if not _empty(getattr(flt, attr, None)):
            raise ValueError(f"query_filter: '{attr}' clauses are not supported (only 'must')")
    must = getattr(flt, "must", None)
    if must is None:
        return []
    if not isinstance(must, (list, tuple)):
        must = [must]
    return [_condition(c, "must") for c in must]


def payload_value(payload, key: str):
    """Value at dotted path ``key`` of a payload (``metadata.source`` -> payload["metadata"]["source"]); _MISSING if
    any step is absent."""
    cur = payload
    for part in key.split("."):
        if not isinstance(cur, dict) or part not in cur:
            return _MISSING
        cur = cur[part]
    return cur


def build_tag_column(payloads: Sequence[dict], key: str, known: dict | None = None):
    """(codes int32 [n], {value_key: code}) for one payload key; -1 where the key is absent (or null).  List- and
    dict-valued fields raise: a multi-valued field cannot be one code per row.  With ``known`` (an existing table, left
    unchanged), its codes are reused and only the values it lacks are returned, numbered after it."""
    codes = np.full(len(payloads), -1, dtype=np.int32)
    base = known or {}
    table: dict = {}
    for i, p in enumerate(payloads):
        v = payload_value(p, key)
        if v is _MISSING or v is None:
            continue
        if isinstance(v, (list, tuple, dict, set)):
            raise ValueError(f"query_filter: payload key {key!r} holds a {type(v).__name__} on row {i}; "
                             "filters on list-valued or nested payload fields are not supported")
        vk = value_key(v)
        codes[i] = base[vk] if vk in base else table.setdefault(vk, len(base) + len(table))
    return codes, table


def _is_number(v) -> bool:
    return isinstance(v, (int, float)) and not isinstance(v, bool)


def build_value_column(payloads: Sequence[dict], key: str) -> np.ndarray:
    """fp64 [n] for one payload key of range filters: the value where it is an int or a float (never a bool), NaN where
    the key is absent, null, NaN or not numeric.  An int beyond 2**53 in magnitude (not exact in fp64) and list- or
    dict-valued fields raise ``ValueError``."""
    vals = np.full(len(payloads), np.nan)
    for i, p in enumerate(payloads):
        v = payload_value(p, key)
        if v is _MISSING or v is None:
            continue
        if isinstance(v, (list, tuple, dict, set)):
            raise ValueError(f"query_filter: payload key {key!r} holds a {type(v).__name__} on row {i}; "
                             "filters on list-valued or nested payload fields are not supported")
        if not _is_number(v):
            continue
        if isinstance(v, int) and abs(v) > EXACT_INT:
            raise ValueError(f"query_filter: payload key {key!r} holds the int {v} on row {i}, beyond 2**53 in "
                             "magnitude: a range filter compares in fp64, which cannot hold it exactly")
        vals[i] = float(v)
    return vals


class PayloadIndex:
    """Per-collection payload index: tag columns (and, for range filters, value columns) built lazily, one per key, on
    the first filter that names the key.  ``payloads`` is the collection's live list: keys indexed later are built from
    its current contents."""

    def __init__(self, payloads: Sequence[dict], load_column, write_codes=None, load_values=None, write_values=None):
        self._payloads = payloads
        self._load = load_column          # load_column(field, codes)
        self._write = write_codes         # write_codes(field, rows, codes): codes of some rows of a loaded column
        self._load_values = load_values   # load_values(field, vals)
        self._write_values = write_values  # write_values(field, rows, vals)
        self.fields: dict[str, tuple[int, dict]] = {}
        self.value_fields: dict[str, int] = {}

    def encode(self, payloads: Sequence[dict]):
        """Codes and values of new payloads for every indexed key, without changing the index: ({key: (codes, new table
        entries)}, {key: values}).  Raises ``ValueError`` (list- or dict-valued field, an int beyond 2**53 under a range
        key) before anything is modified."""
        tags = {}
        for key, (_f, table) in self.fields.items():
            codes, added = build_tag_column(payloads, key, table)
            tags[key] = (codes, added)
        return tags, {key: build_value_column(payloads, key) for key in self.value_fields}

    def apply(self, rows, encoded) -> None:
        """Commit ``encode``'s result for the payloads now stored at ``rows``: new values join their key's table and the
        codes and values are written to the device columns."""
        rows = np.asarray(rows, dtype=np.int64)
        tags, values = encoded
        for key, (codes, added) in tags.items():
            f, table = self.fields[key]
            table.update(added)
            if len(rows):
                self._write(f, rows, codes)
        for key, vals in values.items():
            if len(rows):
                self._write_values(self.value_fields[key], rows, vals)

    def update(self, rows, payloads: Sequence[dict]) -> None:
        """The payloads at ``rows`` changed: codes for every already-indexed key, new values added to its table."""
        self.apply(rows, self.encode(payloads))

    def field(self, key: str):
        if key not in self.fields:
            if len(self.fields) >= MAX_TAG_FIELDS:
                raise ValueError(f"query_filter: at most {MAX_TAG_FIELDS} distinct payload keys can be filtered on "
                                 f"per collection (already indexed: {sorted(self.fields)})")
            codes, table = build_tag_column(self._payloads, key)
            f = len(self.fields)
            self._load(f, codes)
            self.fields[key] = (f, table)
        return self.fields[key]

    def value_field(self, key: str) -> int:
        if key not in self.value_fields:
            if len(self.value_fields) >= MAX_VALUE_FIELDS:
                raise ValueError(f"query_filter: at most {MAX_VALUE_FIELDS} distinct payload keys can be range-filtered "
                                 f"per collection (already indexed: {sorted(self.value_fields)})")
            vals = build_value_column(self._payloads, key)
            f = len(self.value_fields)
            self._load_values(f, vals)
            self.value_fields[key] = f
        return self.value_fields[key]

    def compile_programs(self, filters: Sequence) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """One filter (or None) per query -> (p_off int32 [B+1], prog PRED_DTYPE, pool int32): the postfix programs of
        ``sb_dense_topk_where``.  Every filter is parsed before any column is built, so a refused filter indexes nothing."""
        # one filter object given for many queries (one filter for a whole batch is the common case) is parsed and
        # emitted once; its queries share the steps and the pool codes
        trees = {}
        for f in filters:
            if id(f) not in trees:
                trees[id(f)] = parse_expr(f)
        off = np.zeros(len(filters) + 1, dtype=np.int32)
        prog, pool, span = [], [], {}
        for b, f in enumerate(filters):
            t = trees[id(f)]
            if t is not None:
                if id(f) not in span:
                    s0 = len(prog)
                    self._emit(t, prog, pool)
                    span[id(f)] = (s0, len(prog))
                else:
                    prog.extend(prog[span[id(f)][0]:span[id(f)][1]])
            off[b + 1] = len(prog)
        return off, np.array(prog, dtype=PRED_DTYPE).reshape(-1), np.asarray(pool, dtype=np.int32)

    def _emit(self, node, prog: list, pool: list) -> None:
        kind = node[0]
        if kind == "eq":
            f, table = self.field(node[1])
            code = table.get(value_key(node[2]))
            prog.append((EQ, f, code, 0, 0.0, 0.0, 0, 0) if code is not None else (IN, f, len(pool), 0, 0.0, 0.0, 0, 0))
        elif kind == "any":
            f, table = self.field(node[1])
            codes = sorted({table[value_key(v)] for v in node[2] if value_key(v) in table})   # unknown values drop out
            prog.append((IN, f, len(pool), len(codes), 0.0, 0.0, 0, 0))
            pool.extend(codes)
        elif kind == "range":
            _, key, lo, lo_incl, hi, hi_incl = node
            prog.append((RANGE, self.value_field(key), 0, 0, lo, hi, int(lo_incl), int(hi_incl)))
        else:   # ("and" | "or" | "nor", children) or ("atleast", children, m)
            for c in node[1]:
                self._emit(c, prog, pool)
            op = {"and": AND, "or": OR, "nor": NOR, "atleast": ATLEAST}[kind]
            prog.append((op, 0, len(node[1]), node[2] if kind == "atleast" else 0, 0.0, 0.0, 0, 0))

    def compile(self, filters: Sequence) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """One filter per query -> CSR conditions (f_off [B+1], f_field, f_code); unknown values get code -1."""
        off = np.zeros(len(filters) + 1, dtype=np.int32)
        fields, codes = [], []
        for b, flt in enumerate(filters):
            conds = compile_filter(flt)
            for key, value in conds:
                f, table = self.field(key)
                fields.append(f)
                codes.append(table.get(value_key(value), -1))
            off[b + 1] = off[b] + len(conds)
        return off, np.asarray(fields, dtype=np.int32), np.asarray(codes, dtype=np.int32)


# ------------------------------------------------------------------------------------------------ query_points filters
_REFUSED_CONDITIONS = (("has_id", "HasIdCondition"), ("is_empty", "IsEmptyCondition"), ("is_null", "IsNullCondition"),
                       ("nested", "NestedCondition"))
_REFUSED_FIELDS = ("geo_bounding_box", "geo_radius", "geo_polygon", "values_count", "datetime_range")


def _is_filter(x) -> bool:
    return any(hasattr(x, a) for a in ("must", "should", "must_not", "min_should"))


def _as_list(x) -> list:
    if x is None:
        return []
    return list(x) if isinstance(x, (list, tuple)) else [x]


def _bound(v, key: str, name: str) -> float:
    if not _is_number(v):
        raise ValueError(f"query_filter: Range on {key!r} has a non-numeric {name} bound {v!r} "
                         "(bounds are int or float, never bool)")
    if isinstance(v, int) and abs(v) > EXACT_INT:
        raise ValueError(f"query_filter: Range on {key!r} has the int {name} bound {v}, beyond 2**53 in magnitude "
                         "(not exact in fp64)")
    if v != v:
        raise ValueError(f"query_filter: Range on {key!r} has a NaN {name} bound")
    return float(v)


def _range_node(key: str, r):
    """The bounds given, folded into one (lo, lo_incl, hi, hi_incl); a side without a bound is an inclusive infinity."""
    lo, lo_incl, hi, hi_incl = -np.inf, True, np.inf, True
    gt, gte, lt, lte = (getattr(r, a, None) for a in ("gt", "gte", "lt", "lte"))
    if gte is not None:
        lo, lo_incl = _bound(gte, key, "gte"), True
    if gt is not None:
        v = _bound(gt, key, "gt")
        if v >= lo:
            lo, lo_incl = v, False
    if lte is not None:
        hi, hi_incl = _bound(lte, key, "lte"), True
    if lt is not None:
        v = _bound(lt, key, "lt")
        if v <= hi:
            hi, hi_incl = v, False
    return ("range", key, lo, lo_incl, hi, hi_incl)


def _any_values(vals, key: str) -> list:
    vals = list(vals)
    if len(vals) > MAX_ANY:
        raise ValueError(f"query_filter: MatchAny on {key!r} lists {len(vals)} values (at most {MAX_ANY})")
    if any(isinstance(v, bool) for v in vals):
        raise ValueError(f"query_filter: MatchAny on {key!r} lists a bool (values must be all str or all int)")
    if not (all(isinstance(v, str) for v in vals) or all(isinstance(v, int) for v in vals)):
        raise ValueError(f"query_filter: MatchAny on {key!r} mixes value types (values must be all str or all int)")
    return vals


def _field_node(c, where: str):
    for attr, name in _REFUSED_CONDITIONS:
        if getattr(c, attr, None) is not None:
            raise ValueError(f"query_filter: {name} in {where} is not supported")
    key = getattr(c, "key", None)
    if not isinstance(key, str) or not key:
        raise ValueError(f"query_filter: {where} entry {type(c).__name__} is not a FieldCondition with a key")
    for attr in _REFUSED_FIELDS:
        if getattr(c, attr, None) is not None:
            raise ValueError(f"query_filter: condition on {key!r} uses {attr}, which is not supported")
    m, r = getattr(c, "match", None), getattr(c, "range", None)
    if m is not None and r is not None:
        raise ValueError(f"query_filter: condition on {key!r} has both match and range (give one per condition)")
    if r is not None:
        return _range_node(key, r)
    if m is None:
        raise ValueError(f"query_filter: condition on {key!r} has neither match nor range")
    if getattr(m, "any", None) is not None:
        return ("any", key, _any_values(m.any, key))
    for attr, name in (("except_", "MatchExcept"), ("text", "MatchText"), ("phrase", "MatchPhrase")):
        if getattr(m, attr, None) is not None:
            raise ValueError(f"query_filter: condition on {key!r} uses {name}, which is not supported "
                             "(must_not with MatchAny covers MatchExcept)")
    if not hasattr(m, "value"):
        raise ValueError(f"query_filter: condition on {key!r} uses {type(m).__name__}, which is not supported")
    return ("eq", key, _check_value(m.value, key))


def parse_expr(flt):
    """A ``query_points`` filter -> an expression tree over payload keys, or None for no constraint.  Nodes:
    ("and" | "or" | "nor", [children]), ("atleast", [children], m), ("eq", key, value), ("any", key, [values]),
    ("range", key, lo, lo_incl, hi, hi_incl).  Raises ``ValueError`` naming what is refused or which limit is exceeded."""
    if flt is None:
        return None
    if not _is_filter(flt):
        if hasattr(flt, "key"):   # a bare FieldCondition is the filter must=[condition]
            return ("and", [_field_node(flt, "query_filter")])
        raise ValueError(f"query_filter: unsupported filter object of type {type(flt).__name__}")
    count = [0]

    def filt(f, depth):
        if depth > MAX_DEPTH:
            raise ValueError(f"query_filter: filters nested deeper than {MAX_DEPTH} levels")
        parts = []

        def conds(lst, where):
            out = []
            for c in lst:
                count[0] += 1
                if count[0] > MAX_CONDITIONS:
                    raise ValueError(f"query_filter: more than {MAX_CONDITIONS} conditions in one filter")
                out.append(filt(c, depth + 1) if _is_filter(c) else _field_node(c, where))
            return out

        must = conds(_as_list(getattr(f, "must", None)), "must")
        if must:
            parts.append(("and", must))
        should = conds(_as_list(getattr(f, "should", None)), "should")
        if should:
            parts.append(("or", should))
        must_not = conds(_as_list(getattr(f, "must_not", None)), "must_not")
        if must_not:
            parts.append(("nor", must_not))
        ms = getattr(f, "min_should", None)
        if ms is not None:
            m = getattr(ms, "min_count", None)
            if not isinstance(m, int) or isinstance(m, bool) or m < 0:
                raise ValueError("query_filter: min_should.min_count must be an int >= 0")
            parts.append(("atleast", conds(_as_list(getattr(ms, "conditions", None)), "min_should"), m))
        return parts[0] if len(parts) == 1 else ("and", parts)

    tree = filt(flt, 1)
    if tree == ("and", []):
        return None
    if _stack_depth(tree) > MAX_STACK:
        raise ValueError(f"query_filter: the filter needs more than {MAX_STACK} evaluation stack entries")
    return tree


def _stack_depth(node) -> int:
    if node[0] in ("eq", "any", "range"):
        return 1
    return max([i + _stack_depth(c) for i, c in enumerate(node[1])] + [1])
