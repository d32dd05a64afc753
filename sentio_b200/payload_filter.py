"""Payload filters of the Qdrant search API, compiled for the filtered dense scan (``sb_dense_topk_filtered``).

The reference filters its searches with ``client.search(..., query_filter=_convert_filter(filter))``
(src/core/vector_store/qdrant_store.py:120-146, 351-381); ``_convert_filter`` (:456-471) turns ``{"source": "a.pdf"}``
into ``FieldCondition(key="metadata.source", match=MatchValue(value="a.pdf"))`` and several keys into
``Filter(must=[...])``.  That is the supported subset: a conjunction of "payload key == scalar value" conditions.
Everything else (``should``, ``must_not``, ranges, ``MatchAny``, nested filters, list-valued payload fields, non-scalar
values) raises ``ValueError`` naming the unsupported part -- it is never ignored.

``qdrant_client`` is not a dependency: filters are read by duck typing (``.must``, ``.key``, ``.match.value``), so the
real Qdrant models and any object of the same shape work.
"""
from __future__ import annotations

from typing import Any, Sequence

import numpy as np

MAX_TAG_FIELDS = 16   # SB_MAX_TAG_FIELDS (include/sentio_b200.h)
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


class PayloadIndex:
    """Per-collection payload index: tag columns built lazily, one per key, on the first filter that names the key.
    ``payloads`` is the collection's live list: keys indexed later are built from its current contents."""

    def __init__(self, payloads: Sequence[dict], load_column, write_codes=None):
        self._payloads = payloads
        self._load = load_column          # load_column(field, codes)
        self._write = write_codes         # write_codes(field, rows, codes): codes of some rows of a loaded column
        self.fields: dict[str, tuple[int, dict]] = {}

    def encode(self, payloads: Sequence[dict]):
        """Codes of new payloads for every indexed key, without changing the index: {key: (codes, new table entries)}.
        Raises ``ValueError`` (list- or dict-valued field) before anything is modified."""
        out = {}
        for key, (_f, table) in self.fields.items():
            codes, added = build_tag_column(payloads, key, table)
            out[key] = (codes, added)
        return out

    def apply(self, rows, encoded) -> None:
        """Commit ``encode``'s result for the payloads now stored at ``rows``: new values join their key's table and the
        codes are written to the device column."""
        rows = np.asarray(rows, dtype=np.int64)
        for key, (codes, added) in encoded.items():
            f, table = self.fields[key]
            table.update(added)
            if len(rows):
                self._write(f, rows, codes)

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
