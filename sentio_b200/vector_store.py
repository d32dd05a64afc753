"""B200VectorStore -- an HBM-resident stand-in for the slice of ``qdrant_client.QdrantClient`` the reference uses.

The reference's dense path is ``client.search(collection_name=, query_vector=, limit=, with_payload=True)``
(src/core/retrievers/dense.py:46-64), its cache probe ``client.collection_exists(collection_name=)``
(src/core/retrievers/hybrid.py:101-105) and its BM25 corpus load ``client.scroll(...)``
(src/core/retrievers/factory.py:95-101).  Its store writes with ``client.upsert`` / ``client.delete`` and bootstraps and
inspects collections with ``create_collection(vectors_config=)`` / ``get_collection`` / ``get_collections``
(src/core/vector_store/qdrant_store.py:196-263, 298-349).  This class answers exactly those calls from a ``B200Engine``:
vectors live in HBM as fp16 rows (one engine per collection), payloads / ids stay on the host.  Because it is
call-compatible, the reference's OWN ``DenseRetriever`` runs unchanged on top of it (INTEGRATION.md), and so does ours.

Payload / id schema follows what the reference's ingest writes: ``payload = {"content": text, "metadata": {...}}``,
point id = string (src/core/vector_store/qdrant_store.py:333-340).

Threads: searches may come from a thread pool (the reference's ``retrieve_async``).  Every search (device call plus
its row -> id mapping) and every mutation holds the collection's lock, so a search never maps rows through a
half-updated id / payload mirror.
"""
from __future__ import annotations

import enum
import threading
from types import SimpleNamespace
from dataclasses import dataclass, field
from typing import Any, Sequence

import numpy as np

from .engine import B200Engine
from .payload_filter import PayloadIndex

__all__ = ["B200VectorStore", "ScoredPoint", "Record", "UpdateResult", "CollectionInfo", "Distance", "Datatype",
           "PointGroup", "GroupsResult", "QueryResponse", "RecommendStrategy"]


@dataclass
class ScoredPoint:
    id: Any
    score: float
    payload: dict | None = None
    vector: Any = None
    version: int = 0


@dataclass
class Record:
    id: Any
    payload: dict | None = None
    vector: Any = None


@dataclass
class PointGroup:
    id: Any                 # the group's payload value at ``group_by``
    hits: list = field(default_factory=list)   # its best ScoredPoints, best first


@dataclass
class GroupsResult:
    groups: list = field(default_factory=list)


@dataclass
class QueryResponse:
    points: list = field(default_factory=list)   # ScoredPoints, best first


@dataclass
class UpdateResult:
    status: str = "completed"


class Distance(enum.Enum):
    COSINE = "Cosine"
    DOT = "Dot"
    EUCLID = "Euclid"
    MANHATTAN = "Manhattan"   # accepted by the parser so it can be refused by name: an L1 distance is not a GEMM


class Datatype(enum.Enum):
    """Qdrant's ``VectorParams.datatype``.  FLOAT16 keeps fp16 rows (scores exact on them); FLOAT32 also keeps the
    vectors as given, and every score is exact on them (DESIGN.md K1g); UINT8 keeps integer vectors in [0, 255] at one
    byte per dimension, and every score is exact on them (DESIGN.md K1i)."""
    FLOAT32 = "float32"
    FLOAT16 = "float16"
    UINT8 = "uint8"


class RecommendStrategy(enum.Enum):
    """Qdrant's ``RecommendStrategy`` (DESIGN.md K1j, INTEGRATION.md).  AVERAGE_VECTOR searches avg(P) + (avg(P) - avg(N));
    BEST_SCORE and SUM_SCORES merge the similarities of every row to every example (Cosine and Dot only)."""
    AVERAGE_VECTOR = "average_vector"
    BEST_SCORE = "best_score"
    SUM_SCORES = "sum_scores"


@dataclass
class VectorParams:
    size: int
    distance: Distance = Distance.COSINE
    datatype: Datatype | None = None


@dataclass
class CollectionParams:
    vectors: VectorParams


@dataclass
class CollectionConfig:
    params: CollectionParams


@dataclass
class CollectionInfo:
    points_count: int
    config: CollectionConfig
    status: str = "green"


@dataclass
class CollectionDescription:
    name: str


@dataclass
class CollectionsResponse:
    collections: list = field(default_factory=list)


def _distance_name(dist) -> str:
    return str(getattr(dist, "name", dist))


def parse_distance(dist) -> Distance:
    """A Qdrant distance given as this module's ``Distance``, ``qdrant_client``'s ``Distance`` enum (read by ``.name``)
    or a plain string, case-insensitive ("Cosine", "DOT", "euclid", ...).  Manhattan raises ``ValueError``."""
    name = _distance_name(dist).strip().lower()
    for d in Distance:
        if name in (d.name.lower(), d.value.lower()):
            if d is Distance.MANHATTAN:
                raise ValueError("distance Manhattan is not supported: an L1 distance is not a GEMM "
                                 "(supported: Cosine, Dot, Euclid)")
            return d
    raise ValueError(f"distance {_distance_name(dist)!r} is not supported (supported: Cosine, Dot, Euclid)")


_ENGINE_METRIC = {Distance.COSINE: "cosine", Distance.DOT: "dot", Distance.EUCLID: "euclid"}


def parse_strategy(strategy) -> RecommendStrategy:
    """A recommendation strategy given as this module's ``RecommendStrategy``, ``qdrant_client``'s enum (read by
    ``.name``), its value or a plain string, case-insensitive; ``None`` is AVERAGE_VECTOR, as in Qdrant.  Anything else
    raises ``ValueError``."""
    if strategy is None:
        return RecommendStrategy.AVERAGE_VECTOR
    name = _distance_name(strategy).strip().lower()
    for t in RecommendStrategy:
        if name in (t.name.lower(), t.value):
            return t
    raise ValueError(f"strategy {_distance_name(strategy)!r} is not supported "
                     "(supported: average_vector, best_score, sum_scores)")


def parse_datatype(dt) -> Datatype:
    """A Qdrant vector datatype given as this module's ``Datatype``, ``qdrant_client``'s ``Datatype`` enum (read by
    ``.name``), its value or a plain string, case-insensitive ("float32", "FLOAT16", ...); ``None`` is FLOAT16, this
    store's default.  Any other datatype (int8, bfloat16, ...) raises ``ValueError``."""
    if dt is None:
        return Datatype.FLOAT16
    name = _distance_name(dt).strip().lower()
    for t in Datatype:
        if name in (t.name.lower(), t.value):
            return t
    raise ValueError(f"datatype {_distance_name(dt)!r} is not supported (supported: float32, float16, uint8)")


def _uint8_rows(v: np.ndarray, where: str) -> np.ndarray:
    """The vectors of a UINT8 collection as a uint8 array: every value must be an integer in [0, 255] (NaN, inf,
    fractional and out-of-range values raise ``ValueError``; nothing is rounded)."""
    if v.dtype == np.uint8:
        return v
    f = np.asarray(v, dtype=np.float64)
    ok = np.isfinite(f) & (f >= 0.0) & (f <= 255.0)
    ok &= np.floor(np.where(ok, f, 0.0)) == np.where(ok, f, 0.0)
    if not ok.all():
        bad = tuple(int(i) for i in np.argwhere(~ok)[0])
        raise ValueError(f"{where}: a uint8 collection takes integers in [0, 255]; value {f[bad]!r} at {bad} is not one")
    return f.astype(np.uint8)


class _Collection:
    def __init__(self, name: str, device: int):
        self.name = name
        self.engine = B200Engine(device)
        self.ids: list[Any] = []
        self.payloads: list[dict] = []
        self.row_of: dict[Any, int] = {}
        self.dim = 0
        self.distance = Distance.COSINE
        self.datatype = Datatype.FLOAT16
        self.lock = threading.RLock()
        self._payload_index: PayloadIndex | None = None

    def payload_index(self) -> PayloadIndex:
        # built lazily: a tag column per payload key, on the first filter that names the key
        if self._payload_index is None:
            self._payload_index = PayloadIndex(self.payloads,
                                               lambda f, codes: self.engine.load_dense_tags(f, codes, slot=0),
                                               lambda f, rows, codes: self.engine.dense_tags_write(f, rows, codes, slot=0),
                                               lambda f, vals: self.engine.load_dense_values(f, vals, slot=0),
                                               lambda f, rows, vals: self.engine.dense_values_write(f, rows, vals, slot=0))
        return self._payload_index


_QUERY_KINDS = ("recommend", "discover", "context", "fusion", "order_by", "formula", "sample", "rrf")
MAX_QUERY_DEPTH = 1024   # offset + limit of one query_points request (the engine's top-k bound)


def _query_vector(query, where: str) -> np.ndarray:
    """The vector of a ``query_points`` query: a plain vector or a ``NearestQuery``-shaped object (``.nearest``).  A point
    id, the other query kinds, named or sparse vectors raise ``ValueError``."""
    if query is None:
        raise ValueError(f"{where}: a query vector is required")
    for kind in _QUERY_KINDS:
        if getattr(query, kind, None) is not None:
            raise ValueError(f"{where}: {type(query).__name__} queries are not supported (only nearest-vector queries)")
    if hasattr(query, "nearest"):
        if getattr(query, "mmr", None) is not None:
            raise ValueError(f"{where}: NearestQuery with mmr is not supported (plain nearest-vector queries only)")
        query = query.nearest
    if isinstance(query, (str, int)) or hasattr(query, "hex"):
        raise ValueError(f"{where}: a point id as the query is not supported (give the vector)")
    if isinstance(query, dict) or hasattr(query, "indices"):
        raise ValueError(f"{where}: named, sparse and multi-vector queries are not supported (one dense vector)")
    try:
        q = np.asarray(query, dtype=np.float32)
    except (TypeError, ValueError) as e:
        raise ValueError(f"{where}: the query must be a numeric vector ({e})") from None
    if q.ndim != 1:
        raise ValueError(f"{where}: the query must be one vector, got shape {q.shape}")
    return q


MAX_RECO_EXAMPLES = 256   # examples of one recommendation request (one 256-column block of the scan)


def _reco_example(e, where: str):
    """A recommendation example: a point id (str, int or UUID) or one dense vector (float32)."""
    if isinstance(e, bool):
        raise ValueError(f"{where}: an example must be a point id or a vector, got {e!r}")
    if isinstance(e, (str, int)) or hasattr(e, "hex"):
        return e
    if isinstance(e, dict) or hasattr(e, "indices"):
        raise ValueError(f"{where}: named, sparse and multi-vector examples are not supported (one dense vector)")
    try:
        v = np.asarray(e, dtype=np.float32)
    except (TypeError, ValueError) as err:
        raise ValueError(f"{where}: an example must be a point id or a numeric vector ({err})") from None
    if v.ndim != 1:
        raise ValueError(f"{where}: named, sparse and multi-vector examples are not supported (one dense vector, "
                         f"got shape {v.shape})")
    return v


def _points_columns(points):
    """(ids, vectors, payloads) of a list of ``PointStruct``-shaped objects or a ``Batch``-shaped object."""
    if hasattr(points, "ids") and hasattr(points, "vectors"):
        ids, vecs = list(points.ids), points.vectors
        pls = getattr(points, "payloads", None)
        pls = [None] * len(ids) if pls is None else list(pls)
        if isinstance(vecs, dict):
            raise ValueError("upsert: named vectors are not supported (one unnamed vector per point)")
        vecs = list(vecs)
    else:
        pts = list(points)
        ids = [p.id for p in pts]
        vecs = [p.vector for p in pts]
        pls = [getattr(p, "payload", None) for p in pts]
    if len(vecs) != len(ids) or len(pls) != len(ids):
        raise ValueError("upsert: ids, vectors and payloads must have the same length")
    if any(isinstance(v, dict) for v in vecs):
        raise ValueError("upsert: named vectors are not supported (one unnamed vector per point)")
    return ids, vecs, pls


class B200VectorStore:
    def __init__(self, device: int = 0):
        self._device = device
        self._collections: dict[str, _Collection] = {}

    # ------------------------------------------------------------------ collection management
    def collection_exists(self, collection_name: str) -> bool:
        return collection_name in self._collections

    def create_collection(self, collection_name: str, vectors: np.ndarray | None = None,
                          ids: Sequence[Any] | None = None, payloads: Sequence[dict] | None = None,
                          vectors_config=None, **_ignored) -> None:
        """Upload a whole collection (brute-force search needs no incremental index), or, with Qdrant's
        ``vectors_config=VectorParams(size, distance)`` and no vectors, create an empty one that ``upsert`` fills.
        The distance is Cosine (the default without ``vectors_config``), Dot or Euclid (Qdrant's semantics: Dot scores
        <q, v>, Euclid scores the distance ||q - v|| and ranks it ascending); Manhattan raises ``ValueError``.
        ``vectors_config.datatype``: None or FLOAT16 (this store's default: fp16 rows) or FLOAT32 (the vectors are kept
        as given and every score is exact on them, at 6 bytes per dimension per point in HBM) or UINT8 (integer vectors
        in [0, 255], 1 byte per dimension per point, every score exact on them; other values raise ``ValueError``).  A
        datatype the engine class does not list in ``DATATYPES`` raises ``ValueError``."""
        dist = Distance.COSINE
        dtype = Datatype.FLOAT16
        if vectors_config is not None:
            if isinstance(vectors_config, dict):
                raise ValueError("create_collection: named vectors are not supported (one unnamed vector per point)")
            dist = parse_distance(getattr(vectors_config, "distance", "Cosine"))
            dtype = parse_datatype(getattr(vectors_config, "datatype", None))
        # an engine lists the metrics its load_dense accepts in METRICS; one without the table loads Cosine only
        supported = getattr(B200Engine, "METRICS", {"cosine": 0})
        if _ENGINE_METRIC[dist] not in supported:
            raise ValueError(f"create_collection: distance {dist.value} is not supported by {B200Engine.__name__} "
                             f"(it loads {', '.join(sorted(supported))})")
        # likewise DATATYPES: an engine without the table stores float16 only
        if dtype.value not in getattr(B200Engine, "DATATYPES", {"float16": 0}):
            raise ValueError(f"create_collection: datatype {dtype.value} is not supported by {B200Engine.__name__} "
                             f"(it stores {', '.join(getattr(B200Engine, 'DATATYPES', {'float16': 0}))})")
        if vectors is None:
            if vectors_config is None:
                raise ValueError("create_collection: give vectors or vectors_config")
            vectors = np.zeros((0, int(vectors_config.size)), dtype=np.float32)
        vecs = np.asarray(vectors)
        if dtype is Datatype.UINT8:
            if vecs.ndim != 2:
                raise ValueError("create_collection: vectors must be [n, d]")
            vecs = _uint8_rows(vecs, "create_collection")
        n = vecs.shape[0]
        col = _Collection(collection_name, self._device)
        col.distance = dist
        col.datatype = dtype
        try:
            if dtype in (Datatype.FLOAT32, Datatype.UINT8):
                col.engine.load_dense(vecs, id_base=0, slot=0, metric=_ENGINE_METRIC[dist], storage=dtype.value)
            elif dist is Distance.COSINE:
                col.engine.load_dense(vecs, id_base=0, slot=0)
            else:
                col.engine.load_dense(vecs, id_base=0, slot=0, metric=_ENGINE_METRIC[dist])
        except BaseException:
            col.engine.close()
            raise
        col.ids = list(ids) if ids is not None else [str(i) for i in range(n)]
        col.payloads = list(payloads) if payloads is not None else [{} for _ in range(n)]
        if len(col.ids) != n or len(col.payloads) != n:
            raise ValueError("ids / payloads length must match the number of vectors")
        col.row_of = {pid: i for i, pid in enumerate(col.ids)}
        col.dim = vecs.shape[1]
        old = self._collections.pop(collection_name, None)
        if old is not None:
            old.engine.close()
        self._collections[collection_name] = col

    def delete_collection(self, collection_name: str) -> None:
        col = self._collections.pop(collection_name, None)
        if col is not None:
            col.engine.close()

    def get_collection(self, collection_name: str) -> CollectionInfo:
        col = self._get(collection_name)
        with col.lock:
            return CollectionInfo(points_count=len(col.ids),
                                  config=CollectionConfig(CollectionParams(VectorParams(col.dim, col.distance,
                                                                                        col.datatype))))

    def get_collections(self) -> CollectionsResponse:
        return CollectionsResponse([CollectionDescription(name) for name in list(self._collections)])

    def engine_of(self, collection_name: str) -> B200Engine:
        return self._collections[collection_name].engine

    def locked(self, collection_name: str):
        """The collection's lock (reentrant), for a caller that maps ids to rows (``rows_of``) and then reads those rows
        on the device: held across both, no upsert / delete can move the rows in between."""
        return self._get(collection_name).lock

    def rows_of(self, collection_name: str, ids: Sequence[Any]) -> np.ndarray:
        col = self._collections[collection_name]
        with col.lock:
            return np.asarray([col.row_of.get(i, -1) for i in ids], dtype=np.int64)

    def count(self, collection_name: str) -> int:
        return len(self._collections[collection_name].ids)

    def _get(self, collection_name: str) -> _Collection:
        col = self._collections.get(collection_name)
        if col is None:
            raise ValueError(f"Collection {collection_name} not found")
        return col

    # ------------------------------------------------------------------ writes
    def upsert(self, collection_name: str, points, wait: bool = True, **_ignored) -> UpdateResult:
        """Qdrant ``upsert``: ``points`` is a list of ``PointStruct``-shaped objects (``.id`` / ``.vector`` /
        ``.payload``) or a ``Batch`` (``.ids`` / ``.vectors`` / ``.payloads``).  An existing id overwrites its row
        (vector and payload), a new id appends; within one call the last occurrence of an id wins.  Everything is
        validated before the device is touched, so a ``ValueError`` leaves the collection unchanged.  Always
        synchronous (``wait`` is accepted and ignored)."""
        col = self._get(collection_name)
        ids, vecs, pls = _points_columns(points)
        last = {}
        for i, pid in enumerate(ids):   # first-appearance order, last occurrence's values
            last[pid] = i
        pick = list(last.values())
        uids = list(last)
        if not uids:
            return UpdateResult(status="completed")
        try:
            v = np.asarray([vecs[i] for i in pick], dtype=np.float32)
        except (TypeError, ValueError) as e:
            raise ValueError(f"upsert: vectors must be equal-length numeric sequences ({e})") from None
        if v.ndim != 2 or v.shape[1] != col.dim:
            raise ValueError(f"upsert: vectors must have dimension {col.dim}, got shape {v.shape}")
        if not np.isfinite(v).all():
            raise ValueError("upsert: vectors contain NaN or infinite values")
        if col.datatype is Datatype.UINT8:
            v = _uint8_rows(v, "upsert")
        new_payloads = []
        for i in pick:
            p = pls[i]
            if p is not None and not isinstance(p, dict):
                raise ValueError(f"upsert: payload must be a dict, got {type(p).__name__}")
            new_payloads.append(dict(p) if p is not None else {})
        with col.lock:
            pi = col._payload_index
            encoded = pi.encode(new_payloads) if pi is not None else None
            n0 = len(col.ids)
            rows, appended = [], 0
            for pid in uids:
                r = col.row_of.get(pid)
                if r is None:
                    r = n0 + appended
                    appended += 1
                rows.append(r)
            rows = np.asarray(rows, dtype=np.int64)
            col.engine.dense_upsert(rows, v, slot=0)
            col.ids.extend([None] * appended)
            col.payloads.extend([None] * appended)
            for pid, r, p in zip(uids, rows.tolist(), new_payloads):
                col.ids[r] = pid
                col.payloads[r] = p
                col.row_of[pid] = r
            if pi is not None:
                pi.apply(rows, encoded)
        return UpdateResult(status="completed")

    def delete(self, collection_name: str, points_selector, wait: bool = True, **_ignored) -> UpdateResult:
        """Qdrant ``delete`` by ids: ``points_selector`` is a ``PointIdsList``-shaped object (``.points``) or a plain
        list of ids.  Unknown ids are ignored.  Deleting by filter (``FilterSelector``) raises ``ValueError``."""
        col = self._get(collection_name)
        if hasattr(points_selector, "points"):
            ids = list(points_selector.points)
        elif isinstance(points_selector, (list, tuple)):
            ids = list(points_selector)
        else:   # FilterSelector, a bare Filter, or anything else: never read as a list of ids
            raise ValueError(f"delete: points_selector of type {type(points_selector).__name__} is not supported; "
                             "give PointIdsList(points=[...]) or a list of ids (deleting by filter is not supported)")
        with col.lock:
            rows = sorted({col.row_of[i] for i in ids if i in col.row_of})
            if rows:
                moved_from, moved_to = col.engine.dense_delete(rows, slot=0)
                for r in rows:
                    del col.row_of[col.ids[r]]
                for f, t in zip(moved_from.tolist(), moved_to.tolist()):
                    col.ids[t] = col.ids[f]
                    col.payloads[t] = col.payloads[f]
                    col.row_of[col.ids[t]] = t
                keep = len(col.ids) - len(rows)
                del col.ids[keep:]
                del col.payloads[keep:]   # in place: the payload index reads this list
        return UpdateResult(status="completed")

    def retrieve(self, collection_name: str, ids: Sequence[Any], with_payload: bool = True, with_vectors: bool = False,
                 **_ignored) -> list[Record]:
        """Points by id (unknown ids are skipped, as in Qdrant); vectors are the stored fp16 values, widened (Dot /
        Euclid: c * y, the input to the fp16 precision of its direction).  A FLOAT32 collection returns the vectors as
        given (Cosine: normalised, x / ||x||), as Qdrant does.  A UINT8 collection returns its integer vectors as
        given, for every distance (a normalised uint8 vector does not exist)."""
        col = self._get(collection_name)
        with col.lock:
            rows = [col.row_of[i] for i in ids if i in col.row_of]
            vecs = col.engine.dense_fetch(rows, slot=0) if with_vectors and rows else None
            return [Record(id=col.ids[r], payload=col.payloads[r] if with_payload else None,
                           vector=vecs[j].tolist() if vecs is not None else None) for j, r in enumerate(rows)]

    # ------------------------------------------------------------------ the calls the hot path makes
    def search(self, collection_name: str, query_vector, limit: int = 10, with_payload: bool = True,
               with_vectors: bool = False, query_filter=None, **_ignored) -> list[ScoredPoint]:
        """``query_filter``: a Qdrant ``Filter(must=[FieldCondition(key, match=MatchValue(value))...])`` or a bare
        ``FieldCondition`` (what the reference's ``_convert_filter`` emits): the exact top-``limit`` of the points whose
        payload satisfies every condition.  Other filter shapes raise ``ValueError`` (sentio_b200/payload_filter.py)."""
        col = self._get(collection_name)
        if isinstance(query_vector, tuple):  # ("name", vector) form of the named-vector API
            query_vector = query_vector[1]
        q = np.asarray(query_vector, dtype=np.float32).reshape(1, -1)
        with col.lock:
            limit = max(1, min(int(limit), max(len(col.ids), 1)))   # Qdrant never returns more points than it holds
            filters = self._compile_filters(col, [query_filter]) if query_filter is not None else None
            ids, scores, counts = col.engine.dense_topk(q, int(limit), filters=filters) if filters is not None \
                else col.engine.dense_topk(q, int(limit))
            out = []
            for j in range(int(counts[0])):
                row = int(ids[0, j])
                out.append(ScoredPoint(id=col.ids[row], score=float(scores[0, j]),
                                       payload=col.payloads[row] if with_payload else None))
            return out

    def search_batch(self, collection_name: str, query_vectors, limit: int = 10, with_payload: bool = True,
                     query_filter=None, **_ignored) -> list[list[ScoredPoint]]:
        """``search`` for many query vectors in ONE device batch (the wgmma scan serves 256 queries per HBM pass).
        ``query_filter``: one filter for the whole batch, or a list / tuple with one filter (or None) per query."""
        col = self._get(collection_name)
        q = np.asarray(query_vectors, dtype=np.float32)
        if q.ndim != 2:
            raise ValueError("query_vectors must be [B, d]")
        if q.shape[0] == 0:
            return []
        with col.lock:
            filters = None
            if query_filter is not None:
                per_query = list(query_filter) if isinstance(query_filter, (list, tuple)) else [query_filter] * q.shape[0]
                if len(per_query) != q.shape[0]:
                    raise ValueError(f"query_filter: {len(per_query)} filters for {q.shape[0]} queries")
                if any(f is not None for f in per_query):
                    filters = self._compile_filters(col, per_query)
            ids, scores, counts = col.engine.dense_topk(q, int(limit), filters=filters) if filters is not None \
                else col.engine.dense_topk(q, int(limit))
            return [[ScoredPoint(id=col.ids[int(ids[b, j])], score=float(scores[b, j]),
                                 payload=col.payloads[int(ids[b, j])] if with_payload else None)
                     for j in range(int(counts[b]))] for b in range(q.shape[0])]

    def search_groups(self, collection_name: str, query_vector, group_by: str, limit: int = 10, group_size: int = 1,
                      query_filter=None, with_payload: bool = True, with_vectors: bool = False, with_lookup=None,
                      score_threshold=None, **_ignored) -> GroupsResult:
        """Qdrant ``search_groups``: the best ``limit`` groups of points sharing a payload value at ``group_by`` (a dotted
        path such as ``metadata.parent_id``), ranked by their best point, each with its best ``group_size`` points, over
        the points matching ``query_filter``.  Exact, with the scores and order of ``search``.  Points without the key (or
        with null) are in no group; ``True`` and ``1`` are different groups; a list-valued field raises ``ValueError``.
        ``with_lookup`` and ``score_threshold`` would change the result and are not supported: they raise ``ValueError``."""
        if with_lookup is not None:
            raise ValueError("search_groups: with_lookup is not supported")
        if score_threshold is not None:
            raise ValueError("search_groups: score_threshold is not supported")
        if not isinstance(group_by, str) or not group_by:
            raise ValueError("search_groups: group_by must be a payload key")
        L, G = int(limit), int(group_size)
        if not (1 <= L <= 1024 and 1 <= G <= 1024):
            raise ValueError(f"search_groups: limit {L} and group_size {G} must be in [1, 1024]")
        col = self._get(collection_name)
        if isinstance(query_vector, tuple):  # ("name", vector) form of the named-vector API
            query_vector = query_vector[1]
        q = np.asarray(query_vector, dtype=np.float32).reshape(1, -1)
        with col.lock:
            pi = col.payload_index()
            f, table = pi.field(group_by)
            filters = self._compile_filters(col, [query_filter]) if query_filter is not None else None
            ng, codes, hits, ids, scores = col.engine.dense_groups(q, f, L, G, filters=filters)
            value_of = {c: vk[1] for vk, c in table.items()}
            groups = []
            for g in range(int(ng[0])):
                pts = []
                for r in range(int(hits[0, g])):
                    row = int(ids[0, g, r])
                    pts.append(ScoredPoint(id=col.ids[row], score=float(scores[0, g, r]),
                                           payload=col.payloads[row] if with_payload else None))
                groups.append(PointGroup(id=value_of[int(codes[0, g])], hits=pts))
            return GroupsResult(groups=groups)

    @staticmethod
    def _compile_filters(col: _Collection, filters):
        """CSR conditions for the engine, or None when no query has a condition (the unfiltered search)."""
        off, fld, code = col.payload_index().compile(filters)
        return (off, fld, code) if len(fld) else None

    def query_points(self, collection_name: str, query, query_filter=None, limit: int = 10, offset: int | None = None,
                     score_threshold: float | None = None, with_payload: bool = True, with_vectors: bool = False,
                     using=None, search_params=None, prefetch=None, lookup_from=None, **_ignored) -> QueryResponse:
        """Qdrant ``query_points`` with a nearest-vector query: the exact best points after skipping ``offset``, at most
        ``limit`` of them, over the points matching ``query_filter``.  The filter may use must / should / must_not /
        min_should, nested filters, MatchValue, MatchAny and Range (INTEGRATION.md has the semantics and the refusals).
        ``score_threshold`` keeps scores >= it (Cosine, Dot) or distances <= it (Euclid).  ``with_vectors`` returns
        what ``retrieve`` returns.  ``search_params`` tunes approximate search and is accepted: every search here is
        exact.  A point-id query, other query kinds, ``prefetch``, ``lookup_from``, ``using`` and offset + limit > 1024
        raise ``ValueError``."""
        req = SimpleNamespace(query=query, filter=query_filter, limit=limit, offset=offset,
                              score_threshold=score_threshold, with_payload=with_payload, with_vector=with_vectors,
                              using=using, prefetch=prefetch, lookup_from=lookup_from)
        return self._query(collection_name, [req], "query_points")[0]

    def query_batch_points(self, collection_name: str, requests: Sequence) -> list[QueryResponse]:
        """Qdrant ``query_batch_points``: one ``query_points`` per request (``.query``, ``.filter``, ``.limit``, ``.offset``,
        ``.score_threshold``, ``.with_payload``, ``.with_vector``), answered in ONE device batch of depth max(offset +
        limit).  Each answer is a cut of its query's exact order, so it equals the request run alone."""
        return self._query(collection_name, list(requests), "query_batch_points")

    def _query(self, collection_name: str, reqs: list, where: str) -> list[QueryResponse]:
        col = self._get(collection_name)
        if not reqs:
            return []
        qs, cuts = [], []
        for r in reqs:
            for attr in ("prefetch", "lookup_from", "using"):
                if getattr(r, attr, None) is not None:
                    raise ValueError(f"{where}: {attr} is not supported")
            qs.append(_query_vector(getattr(r, "query", None), where))
            limit = getattr(r, "limit", None)
            limit = 10 if limit is None else limit
            offset = getattr(r, "offset", None) or 0
            if not all(isinstance(v, int) and not isinstance(v, bool) for v in (limit, offset)) or limit < 1 \
                    or offset < 0:
                raise ValueError(f"{where}: limit must be an int >= 1 and offset an int >= 0")
            if offset + limit > MAX_QUERY_DEPTH:
                raise ValueError(f"{where}: offset + limit = {offset + limit} exceeds {MAX_QUERY_DEPTH}")
            # Qdrant's QueryRequest leaves both flags None by default, which it reads as False
            flags = [getattr(r, "with_payload", True), getattr(r, "with_vector", getattr(r, "with_vectors", False))]
            flags = [False if f is None else f for f in flags]
            if not all(isinstance(f, bool) for f in flags):
                raise ValueError(f"{where}: with_payload / with_vector must be True or False (selectors are not "
                                 "supported)")
            t = getattr(r, "score_threshold", None)
            if t is not None and (isinstance(t, bool) or not isinstance(t, (int, float))):
                raise ValueError(f"{where}: score_threshold must be a number")
            cuts.append((offset, limit, t, *flags))
        if len({len(q) for q in qs}) != 1 or len(qs[0]) != col.dim:
            raise ValueError(f"{where}: query vectors must have dimension {col.dim}")
        q = np.stack(qs)
        filters = [getattr(r, "filter", None) for r in reqs]
        with col.lock:
            k = max(1, min(max(o + lim for o, lim, *_ in cuts), max(len(col.ids), 1)))
            if any(f is not None for f in filters):
                programs = col.payload_index().compile_programs(filters)
                ids, scores, counts = col.engine.dense_topk_where(q, k, programs)
            else:
                ids, scores, counts = col.engine.dense_topk(q, k)
            euclid = col.distance is Distance.EUCLID
            out = []
            for b, (offset, limit, t, wp, wv) in enumerate(cuts):
                rows = [int(r) for r in ids[b, offset:min(int(counts[b]), offset + limit)]]
                sc = [float(x) for x in scores[b, offset:offset + len(rows)]]
                if t is not None:   # the order is best first, so the points kept are a prefix
                    keep = sum(1 for x in sc if (x <= t if euclid else x >= t))
                    rows, sc = rows[:keep], sc[:keep]
                vecs = col.engine.dense_fetch(rows, slot=0) if wv and rows else None
                out.append(QueryResponse(points=[
                    ScoredPoint(id=col.ids[r], score=s_, payload=col.payloads[r] if wp else None,
                                vector=vecs[j].tolist() if vecs is not None else None)
                    for j, (r, s_) in enumerate(zip(rows, sc))]))
            return out

    def recommend(self, collection_name: str, positive=None, negative=None, query_filter=None, search_params=None,
                  limit: int = 10, offset: int = 0, with_payload: bool = True, with_vectors: bool = False,
                  score_threshold: float | None = None, using=None, lookup_from=None, strategy=None,
                  **_ignored) -> list[ScoredPoint]:
        """Qdrant ``recommend``: the exact best points "like the positive examples and unlike the negative ones", after
        skipping ``offset``, at most ``limit`` of them, over the points matching ``query_filter`` (the ``query_points``
        filter language).  An example is a point id (its stored vector, as ``retrieve(with_vectors=True)`` returns it) or
        a vector; every id example is left out of the results.  ``strategy`` (None = average_vector):
        average_vector searches avg(P) + (avg(P) - avg(N)) (avg(P) without negatives) with the scores of
        ``query_points``; best_score and sum_scores merge the exact similarities to every example (Cosine and Dot;
        INTEGRATION.md has the formulas).  ``score_threshold`` keeps scores >= it (distances <= it for Euclid
        average_vector).  ``search_params`` is accepted: every search here is exact.  Unknown ids, NaN, wrong
        dimensions, ``using``, ``lookup_from``, no examples, more than 256 of them and offset + limit + id examples
        > 1024 raise ``ValueError`` before anything runs."""
        req = SimpleNamespace(positive=positive, negative=negative, strategy=strategy, filter=query_filter, limit=limit,
                              offset=offset, with_payload=with_payload, with_vector=with_vectors,
                              score_threshold=score_threshold, using=using, lookup_from=lookup_from)
        return self._recommend(collection_name, [req], "recommend")[0]

    def recommend_batch(self, collection_name: str, requests: Sequence) -> list[list[ScoredPoint]]:
        """Qdrant ``recommend_batch``: one ``recommend`` per ``RecommendRequest``-shaped request (``.positive``,
        ``.negative``, ``.strategy``, ``.filter``, ``.limit``, ``.offset``, ``.with_payload``, ``.with_vector``,
        ``.score_threshold``, ``.using``, ``.lookup_from``), answered by one device call per strategy family.  Each
        answer is a cut of its request's exact order, so it equals the request run alone."""
        return self._recommend(collection_name, list(requests), "recommend_batch")

    def _recommend(self, collection_name: str, reqs: list, where: str) -> list[list[ScoredPoint]]:
        col = self._get(collection_name)
        if not reqs:
            return []
        listed = getattr(B200Engine, "RECO_STRATEGIES", {})
        parsed = []
        for r in reqs:
            for attr in ("using", "lookup_from"):
                if getattr(r, attr, None) is not None:
                    raise ValueError(f"{where}: {attr} is not supported")
            strat = parse_strategy(getattr(r, "strategy", None))
            if strat.value not in listed:
                raise ValueError(f"{where}: strategy {strat.value} is not supported by {B200Engine.__name__}")
            if strat is not RecommendStrategy.AVERAGE_VECTOR and col.distance is Distance.EUCLID:
                raise ValueError(f"{where}: strategy {strat.value} is not supported on a Euclid collection "
                                 "(average_vector is)")
            pos = [_reco_example(e, where) for e in (getattr(r, "positive", None) or [])]
            neg = [_reco_example(e, where) for e in (getattr(r, "negative", None) or [])]
            if not pos and not neg:
                raise ValueError(f"{where}: give at least one positive or negative example")
            if strat is RecommendStrategy.AVERAGE_VECTOR and not pos:
                raise ValueError(f"{where}: average_vector needs at least one positive example")
            if len(pos) + len(neg) > MAX_RECO_EXAMPLES:
                raise ValueError(f"{where}: {len(pos) + len(neg)} examples exceed {MAX_RECO_EXAMPLES} per request")
            for v in pos + neg:
                if isinstance(v, np.ndarray):
                    if len(v) != col.dim:
                        raise ValueError(f"{where}: example vectors must have dimension {col.dim}, got {len(v)}")
                    if not np.isfinite(v).all():
                        raise ValueError(f"{where}: an example vector contains NaN or infinite values")
            limit = getattr(r, "limit", None)
            limit = 10 if limit is None else limit
            offset = getattr(r, "offset", None) or 0
            if not all(isinstance(v, int) and not isinstance(v, bool) for v in (limit, offset)) or limit < 1 \
                    or offset < 0:
                raise ValueError(f"{where}: limit must be an int >= 1 and offset an int >= 0")
            flags = [getattr(r, "with_payload", True), getattr(r, "with_vector", getattr(r, "with_vectors", False))]
            flags = [False if f is None else f for f in flags]
            if not all(isinstance(f, bool) for f in flags):
                raise ValueError(f"{where}: with_payload / with_vector must be True or False (selectors are not "
                                 "supported)")
            t = getattr(r, "score_threshold", None)
            if t is not None and (isinstance(t, bool) or not isinstance(t, (int, float))):
                raise ValueError(f"{where}: score_threshold must be a number")
            parsed.append((strat, pos, neg, getattr(r, "filter", None), offset, limit, t, *flags))
        with col.lock:
            # resolve the id examples and check the depth before anything runs
            plans = []
            for strat, pos, neg, flt, offset, limit, t, wp, wv in parsed:
                excl = set()
                for e in pos + neg:
                    if not isinstance(e, np.ndarray):
                        if e not in col.row_of:
                            raise ValueError(f"{where}: no point with id {e!r}")
                        excl.add(col.row_of[e])
                if offset + limit + len(excl) > MAX_QUERY_DEPTH:
                    raise ValueError(f"{where}: offset + limit + id examples = {offset + limit + len(excl)} exceeds "
                                     f"{MAX_QUERY_DEPTH}")
                plans.append((excl, offset + limit + len(excl)))
            id_rows = sorted({r for excl, _ in plans for r in excl})
            stored = dict(zip(id_rows, col.engine.dense_fetch(id_rows, slot=0))) if id_rows else {}

            def vec(e):
                return e if isinstance(e, np.ndarray) else stored[col.row_of[e]]

            results = [None] * len(parsed)
            avg = [b for b, p in enumerate(parsed) if p[0] is RecommendStrategy.AVERAGE_VECTOR]
            merged = [b for b, p in enumerate(parsed) if p[0] is not RecommendStrategy.AVERAGE_VECTOR]
            for group in (avg, merged):
                if not group:
                    continue
                k = max(1, min(max(plans[b][1] for b in group), max(len(col.ids), 1)))
                filters = [parsed[b][3] for b in group]
                programs = col.payload_index().compile_programs(filters) if any(f is not None for f in filters) \
                    else None
                if group is avg:
                    qs = []
                    for b in group:
                        P = np.asarray([vec(e) for e in parsed[b][1]], np.float64)
                        ap = P.sum(0) / len(P)
                        if parsed[b][2]:
                            N = np.asarray([vec(e) for e in parsed[b][2]], np.float64)
                            ap = ap + (ap - N.sum(0) / len(N))
                        qs.append(ap.astype(np.float32))
                    q = np.stack(qs)
                    out = col.engine.dense_topk_where(q, k, programs) if programs is not None \
                        else col.engine.dense_topk(q, k)
                else:
                    ex, r_off, n_pos, strats = [], [0], [], []
                    for b in group:
                        strat, pos, neg = parsed[b][:3]
                        ex.extend(vec(e) for e in pos + neg)
                        r_off.append(len(ex))
                        n_pos.append(len(pos))
                        strats.append(strat.value)
                    out = col.engine.dense_recommend(np.asarray(ex, np.float32), r_off, n_pos, strats, k,
                                                     programs=programs)
                for j, b in enumerate(group):
                    results[b] = tuple(a[j] for a in out)
            euclid = col.distance is Distance.EUCLID
            answers = []
            for (strat, pos, neg, flt, offset, limit, t, wp, wv), (excl, _), (ids, scores, count) in \
                    zip(parsed, plans, results):
                kept = [(int(r), float(s_)) for r, s_ in zip(ids[:int(count)], scores[:int(count)]) if int(r) not in excl]
                kept = kept[offset:offset + limit]
                if t is not None:   # the order is best first, so the points kept are a prefix
                    kept = [(r, s_) for r, s_ in kept if (s_ <= t if euclid else s_ >= t)]
                rows = [r for r, _ in kept]
                vecs = col.engine.dense_fetch(rows, slot=0) if wv and rows else None
                answers.append([ScoredPoint(id=col.ids[r], score=s_, payload=col.payloads[r] if wp else None,
                                            vector=vecs[j].tolist() if vecs is not None else None)
                                for j, (r, s_) in enumerate(kept)])
            return answers

    def search_batch_arrays(self, collection_name: str, query_vectors: np.ndarray, limit: int):
        """Batched extension: (rows [B,k] int64, scores [B,k] float64, counts [B]) without Python objects."""
        col = self._collections[collection_name]
        with col.lock:
            return col.engine.dense_topk(np.asarray(query_vectors, dtype=np.float32), int(limit))

    def scroll(self, collection_name: str, limit: int = 100, offset: int | None = None, with_payload: bool = True,
               with_vectors: bool = False, **_ignored):
        col = self._get(collection_name)
        with col.lock:
            start = int(offset or 0)
            stop = min(len(col.ids), start + int(limit))
            recs = [Record(id=col.ids[i], payload=col.payloads[i] if with_payload else None) for i in range(start, stop)]
            return recs, (stop if stop < len(col.ids) else None)

    def close(self) -> None:
        for col in self._collections.values():
            col.engine.close()
        self._collections.clear()
