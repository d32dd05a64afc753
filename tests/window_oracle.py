"""The error-bounded hand-off window, restated on the CPU (TEST INFRASTRUCTURE, DESIGN.md K1 "Exactness", K1e, K1g, K1i).

Both scans rank rows by an approximate key a(x) with |a(x) - s(x)| <= eps, s(x) the exact key, and re-score in fp64
every row with a >= a_k - 2 eps (a_k: a lower bound of the k-th largest a).  This module restates
  * eps, term by term, as `dense_prep_queries_kernel` computes it (`query_eps`);
  * a(x) up to accumulation error: the key of the rounded operands the scan multiplies, evaluated in fp64
    (`approx_keys`), with the accumulation part of eps as the slack around it;
  * the lower bound of a_k each path uses (`window_bound`): the CUDA-core merge takes the k-th largest list head, the
    wgmma select a radix select over the survivors of the sampled threshold;
and builds corpora on which the window has to do real work (`adversarial_case`, `crowded_case`): baits, rows whose
scan error raises a above their exact key, and decoys, rows with a slightly higher exact key whose error lowers a.  The
exact top-k are then the decoys, the approximate top-k the baits, and the decoys sit between a_k - 2 eps and a_k - eps.

Keys are in the scans' units: the query enters as q^ = q / ||q||.  Cosine: cos(q, x).  Dot: <q^, v>.  Euclid:
r <q^, v> - ||v||^2 / 2 with r = ||q|| (decreasing in ||q - v||).  v is the scored vector: c y for a float16 slot
(metric_oracle), the caller's x for float32 and uint8 slots.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

NUM_SMS = 132          # H100 SXM: CTAs of both scans' persistent grids
MMA_TILE = 128         # dense_mma.cu kTileRows
SAMPLE_ROWS = 16       # dense_mma.cu kSampleRows: rows behind one sampling-pass key
SAMPLE_PER_CTA = 2     # common.cuh dense_sample_per_cta


def f32(v):
    return float(np.float32(v))


def f32_up(v):
    """fp64 -> fp32 rounded upward (__double2float_ru)."""
    r = np.float32(v)
    return float(r) if float(r) >= v else float(np.nextafter(r, np.float32(np.inf)))


def d_pad_of(d, storage):
    return -(-d // (64 if storage == "uint8" else 8)) * (64 if storage == "uint8" else 8)


# --------------------------------------------------------------------------------------------------- eps (dense.cu)
def eps_fp32(d_pad):
    """dense_common.cuh:42 dense_eps_fp32: d_pad 2^-23 + 2^-19."""
    return f32(f32(d_pad * 2.0 ** -23) + 2.0 ** -19)


def eps_mma_acc(d_pad):
    """dense_common.cuh:44 dense_eps_mma_acc: d_pad 2^-22 + 2^-19."""
    return f32(f32(d_pad * 2.0 ** -22) + 2.0 ** -19)


@dataclass
class Bounds:
    """Slot-wide bounds the host keeps (DESIGN.md K1e / K1g / K1i): rho >= max ||v||, hmax >= max ||v||^2 / 2,
    sigma >= max ||y^ - x^|| (Cosine) or ||c y - x|| (Dot / Euclid) on float32 slots."""
    rho: float = 0.0
    hmax: float = 0.0
    sigma: float = 0.0


def prep_query(q, d_pad):
    """(q^ fp32 [d_pad], fp16(q^) [d_pad], ||fp16(q^) - q^||^2, ||q||) as dense.cu:742-771 computes them."""
    qp = np.zeros(d_pad)
    qp[:len(q)] = np.asarray(q, np.float32)
    nrm = float(np.sqrt((qp * qp).sum()))
    qn = (qp / nrm).astype(np.float32) if nrm > 0 else np.zeros(d_pad, np.float32)
    q16 = qn.astype(np.float16)
    e = q16.astype(np.float64) - qn.astype(np.float64)
    return qn, q16, float((e * e).sum()), nrm


def query_eps(q, d_pad, storage, metric, mma, b: Bounds, mutant=None):
    """eps of one query, dense.cu:780-805.  mutant: None, "M1" (no query-rounding term, dense.cu:781), "M3" (no rho,
    :789), "M4" (Euclid without r, :797), "M5" (no sigma, :784 / :790 / :798)."""
    _, _, t, nrm = prep_query(q, d_pad)
    zero = not nrm > 0
    sigma = 0.0 if mutant == "M5" else b.sigma
    e = 0.0
    if not zero:   # dense.cu:781
        e = f32(f32(np.sqrt(t) * 1.0001 if mutant != "M1" else 0.0) + eps_mma_acc(d_pad)) if mma else eps_fp32(d_pad)
    if storage == "float32" and metric == "cosine" and not zero:   # dense.cu:784
        e = f32_up(e + sigma)
    if metric == "cosine":
        return e
    ed = (e + 2.0 ** -20) * (b.rho if mutant != "M3" else 1.0) * 1.001   # dense.cu:789
    if storage == "float32":
        ed += sigma                                                        # dense.cu:790
    if metric == "dot":
        return 0.0 if zero else f32_up(ed)                                 # dense.cu:793
    rr = 0.0 if zero else f32(nrm)
    ee = ((rr if mutant != "M4" else 1.0) * ed + (rr * b.rho + b.hmax) * 2.0 ** -20) * 1.001   # dense.cu:797
    if storage == "float32":
        ee += b.rho * sigma * 1.001                                        # dense.cu:798
    return f32_up(ee)


def euclid_resolves(q, b: Bounds, eps):
    """dense.cu:801-802: the query is answered by the scans (not routed to the fp64 brute force up front)."""
    rr = f32(np.linalg.norm(np.asarray(q, np.float64)))
    res = (rr + b.rho) ** 2 * 2.0 ** -41
    return res * 1024.0 <= eps


# ------------------------------------------------------------------------------------------ the stored representation
@dataclass
class Slot:
    """What a slot keeps of input rows x (dense.cu store kernels; metric_oracle / f32_oracle / u8_oracle)."""
    storage: str
    metric: str
    x: np.ndarray                     # the caller's rows (float32 or uint8)
    y: np.ndarray = None              # fp16 rows the fp16 scans read (float16 and float32 storage)
    c: np.ndarray = None              # Dot / Euclid: v = c y
    scale: np.ndarray = None          # per-row scan scale (inv_norm)
    h: np.ndarray = None              # Euclid: ||v||^2 / 2 rounded up to fp32
    v: np.ndarray = None              # the exactly scored vectors, fp64


def make_slot(x, storage, metric):
    s = Slot(storage, metric, x)
    if storage == "uint8":
        v = x.astype(np.float64)
        ss = (v * v).sum(axis=1)
        s.v = v
        s.scale = np.where(ss > 0, (1.0 / np.sqrt(np.where(ss > 0, ss, 1.0))).astype(np.float32), 0.0) \
            if metric == "cosine" else np.ones(len(x))
        s.h = np.array([f32_up(0.5 * t) for t in ss]) if metric == "euclid" else np.zeros(len(x))
        return s
    x64 = x.astype(np.float32).astype(np.float64)
    nrm = np.sqrt((x64 * x64).sum(axis=1))
    y = (x64 / np.where(nrm > 0, nrm, 1.0)[:, None]).astype(np.float16)
    y64 = y.astype(np.float64)
    ss16 = (y64 * y64).sum(axis=1)
    s.y = y
    if metric == "cosine":
        s.scale = np.where(ss16 > 0, (1.0 / np.sqrt(np.where(ss16 > 0, ss16, 1.0))).astype(np.float32), 0.0)
        s.h = np.zeros(len(x))
        s.c = None
        s.v = x64 if storage == "float32" else y64
        return s
    c = np.divide(nrm, np.sqrt(ss16), out=np.zeros(len(x)), where=ss16 > 0)
    s.c = c
    s.scale = c.astype(np.float32).astype(np.float64)
    s.h = np.array([f32_up(0.5 * cc * cc * t) for cc, t in zip(c, ss16)]) if metric == "euclid" else np.zeros(len(x))
    s.v = x64 if storage == "float32" else c[:, None] * y64
    return s


def slot_bounds(slot: Slot):
    """rho, hmax, sigma as a load sets them (DESIGN.md K1e, K1g, K1i), with the load's widening."""
    v = slot.v
    nv = np.sqrt((v * v).sum(axis=1))
    b = Bounds()
    if slot.metric != "cosine":
        b.rho = float(nv.max()) * (1.0 + 2.0 ** -20)
        b.hmax = float(slot.h.max()) if slot.metric == "euclid" else 0.0
    if slot.storage == "float32":
        x64 = slot.x.astype(np.float64)
        y64 = slot.y.astype(np.float64)
        if slot.metric == "cosine":
            xn = np.sqrt((x64 * x64).sum(axis=1, keepdims=True))
            yn = np.sqrt((y64 * y64).sum(axis=1, keepdims=True))
            dlt = y64 / np.where(yn > 0, yn, 1.0) - x64 / np.where(xn > 0, xn, 1.0)
            m = 1.0
        else:
            dlt = slot.c[:, None] * y64 - x64
            m = nv
        sg = np.sqrt((dlt * dlt).sum(axis=1))
        b.sigma = float((sg * (1 + 2.0 ** -39) + m * 2.0 ** -39).max())
    return b


def merge_bounds(a: Bounds, b: Bounds):
    """An upsert only raises the bounds (dense.cu:2473-2475)."""
    return Bounds(max(a.rho, b.rho), max(a.hmax, b.hmax), max(a.sigma, b.sigma))


# ---------------------------------------------------------------------------------------------- keys a(x) and s(x)
def exact_keys(slot: Slot, q):
    """s(x) in fp64 on the scored vectors."""
    q64 = np.asarray(q, np.float32).astype(np.float64)
    nq = float(np.sqrt(q64 @ q64))
    v = slot.v
    dot = v @ q64
    if slot.metric == "cosine":
        den = np.sqrt((v * v).sum(axis=1)) * nq
        return np.divide(dot, den, out=np.zeros(len(v)), where=den > 0)
    if slot.metric == "dot":
        return dot / nq
    return dot - 0.5 * (v * v).sum(axis=1)


def approx_keys(slot: Slot, q, mma, b: Bounds):
    """(a, slack): the scan key of every row, evaluated in fp64 on the operands the scan multiplies -- fp16(q^) and the
    stored fp16 / uint8 row on the wgmma scan, the fp32 q^ and the fp16 row on the CUDA-core scan -- times the row's
    scale; slack = the accumulation part of eps (eps of an exactly representable query on a float16 slot), which
    bounds how far the device's fp32 sums and roundings can move the key from it."""
    d_pad = d_pad_of(slot.x.shape[1], slot.storage)
    qn, q16, _, nrm = prep_query(q, d_pad)
    op = (q16 if mma else qn).astype(np.float64)[:slot.x.shape[1]]
    rows = slot.v if slot.storage == "uint8" else slot.y.astype(np.float64)
    a = (rows @ op) * slot.scale
    if slot.metric == "euclid":
        a = f32(nrm) * a - slot.h
    slack = query_eps(q, d_pad, "float16", slot.metric, mma, Bounds(b.rho, b.hmax, 0.0), mutant="M1")
    return a, slack


def composite_keys(a, rows):
    """The scans' 64-bit keys (common.cuh make_key32): orderable fp32 score above ~row (lower rows win ties)."""
    def orderable(f):
        u = np.asarray(f, np.float32).view(np.uint32).astype(np.uint64)
        return np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)
    keys = (orderable(a) << np.uint64(32)) | (~np.asarray(rows, np.uint64) & np.uint64(0xFFFFFFFF))
    return keys


def select_lb(a, rows, k):
    """The wgmma select's lower bound of the k-th largest key among survivors (a, rows), dense_mma.cu:484-507:
    MSB-first 8-bit digits of the composite key, stopping once the bucket of the k-th key holds <= 16 keys; the score
    field of the prefix (undecided bits zero)."""
    keys = composite_keys(a, rows)
    if len(keys) <= k:
        return -np.inf
    prefix, mask, need = 0, 0, k
    for shift in range(56, -1, -8):
        sel = keys[(keys & np.uint64(mask)) == np.uint64(prefix)]
        dg = ((sel >> np.uint64(shift)) & np.uint64(0xff)).astype(np.int64)
        hist = np.bincount(dg, minlength=256)
        acc = 0
        for b in range(255, -1, -1):   # descending digits
            if acc + hist[b] >= need:
                need -= acc
                prefix |= b << shift
                bucket = int(hist[b])
                break
            acc += hist[b]
        mask |= 0xff << shift
        if bucket <= 16:
            break
    hi = (prefix >> 32) & 0xFFFFFFFF
    u = np.uint32(hi & 0x7FFFFFFF) if hi & 0x80000000 else np.uint32(~hi & 0xFFFFFFFF)
    return float(np.array([u], np.uint32).view(np.float32)[0])


def window_bound(a, k, eps, mma, n, match=None, sample_all=None):
    """The device's lower bound of a_k for keys a of rows 0..n-1 (match: the filter's matching rows).
    wgmma: sampling pass (every tile sampled: n_pad / 128 <= 2 x 132) -> threshold (k-th best 16-row maximum) - 2 eps
    -> survivors -> radix select.  ``sample_all`` ignores the match bits in the sampling maxima (mutant M7).
    CUDA-core: the k-th largest of the heads of the per-CTA lists (32-row tiles dealt round-robin to the CTAs)."""
    live = np.ones(n, bool) if match is None else np.asarray(match, bool)
    a = np.asarray(a, np.float64)
    n_pad = -(-n // 128) * 128
    if mma:
        assert n_pad // MMA_TILE <= SAMPLE_PER_CTA * NUM_SMS, "corpus too large for the every-tile-sampled restatement"
        g = np.full(n_pad, -np.inf)
        g[:n] = np.where(live | bool(sample_all), a, -np.inf)
        maxima = g.reshape(-1, SAMPLE_ROWS).max(axis=1)
        thr = -np.inf if len(maxima) <= k else np.sort(maxima)[::-1][k - 1] - 2 * eps
        surv = np.flatnonzero(live & (a >= thr))
        return select_lb(a[surv], surv, k), thr
    tile = 32                                 # 8 consumer warps x 4 rows (d_pad <= 256)
    tiles = n_pad // tile
    grid = min(NUM_SMS, tiles)
    kp = max(128, 1 << (k + 28 - 1).bit_length())
    heads_per = -(-kp // grid)
    cta = (np.arange(n) // tile) % grid
    heads = []
    for c in range(grid):
        m = np.flatnonzero((cta == c) & live)
        heads.extend(np.sort(a[m])[::-1][:heads_per])
    heads = np.sort(np.asarray(heads))[::-1]
    return (heads[k - 1] if len(heads) >= k else -np.inf), -np.inf


# ------------------------------------------------------------------------------------------------------- analysis
@dataclass
class Verdict:
    exact_top: np.ndarray      # exact top-k rows
    approx_differs: bool       # (a): some exact top-k row is outside the approximate top-k whatever the accumulation
    kept: bool                 # (b): the true eps keeps every exact top-k row inside the window
    missed: bool               # (c): the mutant leaves some exact top-k row outside the window (or below the threshold)
    margin_kept: float         # (b)'s margin in units of eps
    margin_missed: float       # (c)'s margin in units of eps


def analyse(slot: Slot, q, k, mma, b: Bounds, mutant=None, b_mut: Bounds = None, match=None):
    """(a), (b) and (c) for one query, with every key anywhere inside [a - slack, a + slack]."""
    n = len(slot.x)
    d_pad = d_pad_of(slot.x.shape[1], slot.storage)
    s = exact_keys(slot, q)
    a, slack = approx_keys(slot, q, mma, b)
    rows = np.arange(n) if match is None else np.flatnonzero(match)
    top = rows[np.lexsort((rows, -s[rows]))[:k]]
    eps = query_eps(q, d_pad, slot.storage, slot.metric, mma, b)
    lo, hi = a - slack, a + slack
    kth_lo = np.sort(lo[rows])[::-1][k - 1]
    approx_differs = bool(hi[top].min() < kth_lo)
    # (b): the bound of a_k never exceeds the k-th largest key; the window's lower edge is at most kth_hi - 2 eps
    kth_hi = np.sort(hi[rows])[::-1][k - 1]
    margin_kept = (lo[top].min() - (kth_hi - 2 * eps)) / eps
    # (c)
    missed, margin_missed = False, float("nan")
    if mutant is not None:
        eps_m = query_eps(q, d_pad, slot.storage, slot.metric, mma, b_mut or b,
                          mutant=mutant if mutant in ("M1", "M3", "M4", "M5") else None)
        factor = 1.0 if mutant == "M2" else 2.0
        lb, thr = window_bound(a, k, eps_m, mma, n, match=match, sample_all=(mutant == "M7"))
        # the bound is 1-Lipschitz in the keys: every key moving by <= slack moves it by <= slack
        # a row is lost below the window's edge or below the full pass's threshold (M7: that of the unmasked maxima)
        edge = max(lb - slack - factor * eps_m, thr - slack)
        margin_missed = (edge - hi[top].min()) / eps
        missed = bool(margin_missed > 0)
    return Verdict(top, approx_differs, bool(margin_kept >= 0), missed, float(margin_kept), margin_missed)


# ------------------------------------------------------------------------------------------------------ generators
D = 64                 # dimension of every case: small, so a 4-sparse query's fp16 rounding is a large part of eps
SUPPORT = 4            # non-zeros of an adversarial query; query m uses coordinates 4 m .. 4 m + 3
N_ADV = 3              # adversarial queries per case
FREE = np.arange(SUPPORT * N_ADV, D)   # coordinates no adversarial query reads


def band_row(m, j):
    """Row of band member j of adversarial query m: 32-row CUDA-core tile j (its CTA is j mod 132, so the k baits
    j < k head k distinct lists), a 16-row wgmma sampling group of its own for every j."""
    return 32 * j + 8 * m


@dataclass
class Case:
    name: str
    storage: str
    metric: str
    x: np.ndarray                  # the rows a search sees (after the upsert, if any)
    q: np.ndarray                  # [B_max, D] queries: the N_ADV adversarial queries, repeated
    k: int
    scans: tuple                   # "mma" (wgmma, B = 16 and 256) and / or "core" (CUDA-core, mode 1, B = 3)
    mutants: tuple                 # mutants each scan listed must fail
    bounds: Bounds = None          # slot bounds the search uses
    x0: np.ndarray = None          # upsert cases: the background loaded first ...
    up_rows: np.ndarray = None     # ... then these rows overwritten with x[up_rows]
    bounds0: Bounds = None         # the bounds of the background alone (mutant M6)
    match: np.ndarray = None       # filtered: the rows matching every query's condition (tag 1)
    bands: list = field(default_factory=list)   # per adversarial query: (decoy rows, bait rows)


def _unit(v):
    return v / np.linalg.norm(v)


def _query(rng, m, kind):
    """Adversarial query m: a 4-sparse positive query.  "rounded": the one of 400 random tries whose rounding error
    fp16(q^) - q^ (the wgmma scan's) has the largest part orthogonal to q^; "exact": q^ = (1/2, 1/2, 1/2, 1/2), exact in fp16 (no query rounding:
    the error is the row's, sigma)."""
    q = np.zeros(D, np.float32)
    sl = slice(SUPPORT * m, SUPPORT * (m + 1))
    if kind == "exact":
        q[sl] = 1.0
        return q
    best, best_t = None, -1.0
    for _ in range(400):
        c = np.zeros(D, np.float32)
        c[sl] = rng.uniform(0.3, 1.0, SUPPORT).astype(np.float32)
        qn, q16, _, _ = prep_query(c, D)
        e = q16.astype(np.float64) - qn
        t = e @ e - (e @ qn) ** 2 / (qn.astype(np.float64) @ qn)   # the part orthogonal to q^ tells rows apart
        if t > best_t:
            best, best_t = c, t
    return best


def _directions(rng, m, q, n, alpha, beta, nonneg):
    """n unit rows alpha q^ + beta p + gamma w: p the unit part of q's fp16 rounding error orthogonal to q^ (any unit
    vector orthogonal to q^ in the support when the query is exact), w random on the free coordinates."""
    qh = np.asarray(q, np.float64) / np.linalg.norm(q)
    _, q16, _, _ = prep_query(q, D)
    e = q16.astype(np.float64) - qh
    p = e - (e @ qh) * qh
    if np.linalg.norm(p) < 1e-12:
        p = np.zeros(D)
        p[SUPPORT * m:SUPPORT * (m + 1)] = [1.0, -1.0, 1.0, -1.0]
        p -= (p @ qh) * qh
    p = _unit(p)
    w = np.zeros((n, D))
    w[:, FREE] = np.abs(rng.standard_normal((n, len(FREE)))) if nonneg else rng.standard_normal((n, len(FREE)))
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    g = np.sqrt(np.maximum(0.0, 1.0 - alpha ** 2 - beta ** 2))
    return alpha[:, None] * qh[None, :] + beta[:, None] * p[None, :] + g[:, None] * w


def _rows(u, norm, storage):
    if storage == "uint8":
        return np.clip(np.rint(u * norm), 0, 255).astype(np.uint8)
    return (u * norm).astype(np.float32)


def _background(rng, n, storage, norm, kind):
    if kind == "eighths":      # +-1/8: norm exactly 1, every component exact in fp16 (sigma = 0 on a float32 slot)
        return (rng.choice([-0.125, 0.125], (n, D)) * norm).astype(np.float32)
    if kind == "bits":         # uint8 rows of zeros and ones: small norms
        return rng.integers(0, 2, (n, D)).astype(np.uint8)
    u = rng.standard_normal((n, D))
    u[:, :SUPPORT * N_ADV] *= 0.1
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    if storage == "uint8":
        return np.clip(np.rint(np.abs(u) * norm * 0.3), 0, 255).astype(np.uint8)
    return (u * norm).astype(np.float32)


def _key_scale(metric, norm, r):
    """d(exact key) / d(alpha) for rows of the given norm: the s-units of one unit of cosine."""
    return 1.0 if metric == "cosine" else (norm if metric == "dot" else r * norm)


def _select_band(rng, storage, metric, q, m, k, mma, norm, r, s0, bounds_hint, nonneg, beta_max):
    """(decoy rows, bait rows) for adversarial query m: k candidate rows just above s0 whose scan error lowers a the
    most, and k just below whose error raises it the most."""
    ks = _key_scale(metric, norm, r)
    probe = _directions(rng, m, q, 4000, np.full(4000, s0), rng.uniform(-beta_max, beta_max, 4000), nonneg)
    sl = make_slot(_rows(probe, norm, storage), storage, metric)
    a, _ = approx_keys(sl, q * (r if metric == "euclid" else 1.0), mma, bounds_hint)
    err = a - exact_keys(sl, q * (r if metric == "euclid" else 1.0))
    gap = float(np.quantile(err, 0.98) - np.quantile(err, 0.02))
    # integer rows scatter s far more than the band is wide: a wider band (the uint8 cases target M1, whose eps loses
    # almost all of its width) and a larger pool
    delta, width = (0.1 * gap, 0.04 * gap) if storage != "uint8" else (0.1 * gap, 0.3 * gap)
    s_mid = s0 if metric == "cosine" else float(np.median(exact_keys(sl, q * (r if metric == "euclid" else 1.0))))
    n = 40000 if storage != "uint8" else 160000
    alpha = s0 + rng.uniform(-width - 0.02 * gap, delta + width + 0.02 * gap, n) / ks
    u = _directions(rng, m, q, n, alpha, rng.uniform(-beta_max, beta_max, n), nonneg)
    x = _rows(u, norm, storage)
    sl = make_slot(x, storage, metric)
    qq = q * (r if metric == "euclid" else 1.0)
    s = exact_keys(sl, qq)
    a, _ = approx_keys(sl, qq, mma, bounds_hint)
    err = a - s
    base = s_mid
    lowr = np.flatnonzero((s >= base - width) & (s < base))
    high = np.flatnonzero((s >= base + delta) & (s < base + delta + width))
    assert len(lowr) >= k and len(high) >= k, "candidate pool too small"
    baits = lowr[np.argsort(-err[lowr])[:k]]
    decoys = high[np.argsort(err[high])[:k]]
    return x[decoys], x[baits]


CASES = {
    # name: (storage, metric, scans, mutants, query kind, band norm, query norm r, background, upsert)
    "f16_cosine": ("float16", "cosine", ("mma",), ("M1", "M2"), "rounded", 1.0, 1.0, "random", False),
    "f16_dot": ("float16", "dot", ("mma",), ("M1", "M2", "M3"), "rounded", 1e3, 1.0, "random", False),
    "f16_euclid": ("float16", "euclid", ("mma",), ("M1", "M2", "M4"), "rounded", 1.0, 1e2, "random", False),
    "f32_cosine": ("float32", "cosine", ("mma", "core"), ("M5",), "exact", 1.0, 1.0, "random", False),
    "f32_dot": ("float32", "dot", ("mma", "core"), ("M5",), "exact", 1.0, 1.0, "random", False),
    "f32_euclid": ("float32", "euclid", ("mma", "core"), ("M5",), "exact", 1.0, 1.0, "random", False),
    "upsert_f32_cosine": ("float32", "cosine", ("mma", "core"), ("M6",), "exact", 1.0, 1.0, "eighths", True),
    "upsert_f16_dot": ("float16", "dot", ("mma",), ("M6",), "rounded", 1e3, 1.0, "eighths", True),
    "upsert_u8_dot": ("uint8", "dot", ("mma",), ("M6",), "rounded", 400.0, 1.0, "bits", True),
    "u8_cosine": ("uint8", "cosine", ("mma",), ("M1",), "rounded", 400.0, 1.0, "random", False),
    "u8_dot": ("uint8", "dot", ("mma",), ("M1",), "rounded", 400.0, 1.0, "random", False),
    "filtered_f32_cosine": ("float32", "cosine", ("mma", "core"), ("M7",), "exact", 1.0, 1.0, "random", False),
}
N_ROWS = 12000         # > 8192 (the wgmma scan is eligible), <= 2 x 132 tiles of 128 (every tile sampled)
K = 100
B_MAX = 256


def adversarial_case(name, seed=0):
    storage, metric, scans, mutants, qkind, norm, r, bg, upsert = CASES[name]
    rng = np.random.default_rng(seed + sum(map(ord, name)))
    x = _background(rng, N_ROWS, storage, 1.0 if storage != "uint8" else 100.0, bg)
    x0 = x.copy()
    q = rng.standard_normal((B_MAX, D)).astype(np.float32)
    if storage == "uint8":
        q = np.abs(q)
    mma = "mma" in scans
    beta_max = 0.85 if storage != "uint8" else 0.35
    bands, up_rows = [], []
    hint = Bounds(rho=norm * (1 + 2.0 ** -20), hmax=0.5 * norm * norm * 1.001)
    for m in range(N_ADV):
        qm = _query(rng, m, qkind)
        q[m] = qm / np.linalg.norm(qm) * (r if metric == "euclid" else 1.0)
        decoys, baits = _select_band(rng, storage, metric, q[m] / np.linalg.norm(q[m]), m, K, mma, norm, r, 0.5,
                                     hint, storage == "uint8", beta_max)
        rows_b = np.asarray([band_row(m, j) for j in range(K)])
        rows_d = np.asarray([band_row(m, j) for j in range(K, 2 * K)])
        x[rows_b] = baits
        x[rows_d] = decoys
        bands.append((rows_d, rows_b))
        up_rows += list(rows_b) + list(rows_d)
    q[N_ADV:] = q[np.arange(N_ADV, B_MAX) % N_ADV]   # a batch of any size is made of the adversarial queries
    match = None
    if name.startswith("filtered"):
        match = np.arange(N_ROWS) % 2 == 0
        for rows_d, rows_b in bands:
            match[rows_d] = match[rows_b] = True
        hi_rows = np.arange(N_ROWS // 16) * 16 + 15
        for m in range(N_ADV):     # above every bait, but outside the filter: the sampling maxima must skip them
            sel = hi_rows[hi_rows // 16 % N_ADV == m]
            qh = q[m] / np.linalg.norm(q[m])
            x[sel] = _rows(_directions(rng, m, qh, len(sel), np.full(len(sel), 0.9), np.zeros(len(sel)), False),
                           norm, storage)
            match[sel] = False
    slot = make_slot(x, storage, metric)
    case = Case(name, storage, metric, x, q, K, scans, mutants, bounds=slot_bounds(slot), match=match, bands=bands)
    if upsert:
        case.x0 = x0
        case.up_rows = np.asarray(sorted(up_rows))
        case.bounds0 = slot_bounds(make_slot(x0, storage, metric))
        case.bounds = merge_bounds(case.bounds0, slot_bounds(make_slot(x[case.up_rows], storage, metric)))
    return case


def mma_list_capacity(n, k):
    """dense_mma.cu:612-640, unfiltered: the per-(CTA, query) survivor list capacity of the full pass."""
    total_tiles = -(-n // 128)
    grid = min(NUM_SMS, total_tiles)
    per_cta = max(SAMPLE_PER_CTA, min(8, (4 * k // 8 + grid - 1) // grid))
    sample_tiles = min(per_cta * grid, total_tiles)
    sgrid = min(grid, sample_tiles)
    worst = ((total_tiles + grid - 1) // grid + 1) * 128
    samp_keys = ((sample_tiles + sgrid - 1) // sgrid + 1) * 8
    f = k / (8.0 * sample_tiles)
    pss = 1.0 if f >= 0.95 else -np.log(1.0 - f) / 16.0
    expect = int(worst * pss) + 1
    return min(worst, max(8 * expect + 256, samp_keys))


CROWD_N = 40000        # 313 wgmma tiles: CTAs 0 .. 48 scan three (rows of tiles c, c + 132, c + 264)


def crowded_rows():
    """Every row of wgmma CTA 0 (384 rows: more than its survivor list holds) plus two more 32-row tiles of CUDA-core
    CTA 0 (160 rows of one CTA: more than its 128-entry list)."""
    r = [np.arange(t * 128, t * 128 + 128) for t in (0, 132, 264)]
    r += [np.arange(t * 32, t * 32 + 32) for t in (132, 264)]
    return np.concatenate(r)


def crowded_case(seed=0):
    """A cluster of exact duplicates crowding one CTA of each scan, on top for the adversarial queries: the whole
    cluster is inside the window, so a list fills with window rows and the query must take the exact fallback."""
    rng = np.random.default_rng(seed + 7)
    x = _background(rng, CROWD_N, "float16", 1.0, "random")
    u0 = _unit(rng.standard_normal(D))
    rows = crowded_rows()
    x[rows] = u0.astype(np.float32)
    q = rng.standard_normal((B_MAX, D)).astype(np.float32)
    q[:N_ADV] = (u0[None, :] + 0.05 * rng.standard_normal((N_ADV, D))).astype(np.float32)
    return x, q, rows
