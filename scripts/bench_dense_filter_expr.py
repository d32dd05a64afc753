#!/usr/bin/env python
"""Boolean payload filters (sb_dense_topk_where, DESIGN.md K1h) at bench scale: 1 M x 1024 synthetic corpus (the seeds
of bench.py), 256-query batches, k = 100.

(a) bench_dense_filter.py's fractions (100 %, 10 %, 1 %, 0.1 %, 0.01 % of the rows match one tag value), each step
    alternating the legacy conjunction entry (sb_dense_topk_filtered) with the same filter as a program
    (sb_dense_topk_where): queries/s of both and the mask time per call of each.
(b) shaped filters through the program entry: `should` of 3 values, must + must_not, Range at ~50 %, 1 % and 0.05 %,
    MatchAny of 10 and of 1000 values, a nested filter.  Per filter: queries/s of the device call on precompiled
    programs, the host time of compiling the batch's 256 filters (PayloadIndex.compile_programs, which every
    query_batch_points call pays before the device call), mask / scan / gather ms per call, an 8-query fp64 oracle check
    and the fallback count.

The card's name and power limit are read in the same run.  Prints one JSON line (and writes it with --out).

    python scripts/bench_dense_filter_expr.py [--n-docs 1000000] [--dim 1024] [--steps 10] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import sys
import time
from types import SimpleNamespace as NS

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from bench_dense_filter import FRACTIONS, card, oracle_topk   # noqa: E402


def _fc(key, **m):
    return NS(key=key, match=NS(**m), range=None)


def _rg(key, **b):
    r = NS(gt=None, gte=None, lt=None, lte=None)
    for k, v in b.items():
        setattr(r, k, v)
    return NS(key=key, range=r, match=None)


SHAPED = {
    "should_3_values": NS(should=[_fc("src", value=f"s{i}") for i in (1, 2, 3)]),
    "must_and_must_not": NS(must=[_fc("tenant", value="A")], must_not=[_fc("src", any=[f"s{i}" for i in range(10)])]),
    "range_50pct": NS(must=[_rg("price", lt=0.5)]),
    "range_1pct": NS(must=[_rg("price", gte=0.25, lt=0.26)]),
    "range_0.05pct": NS(must=[_rg("price", gt=0.9, lte=0.9005)]),
    "match_any_10": NS(must=[_fc("tag", any=list(range(0, 10000, 1000)))]),
    "match_any_1000": NS(must=[_fc("tag", any=list(range(0, 10000, 10)))]),
    "nested": NS(must=[NS(should=[_rg("year", gte=2023), NS(must=[_fc("tenant", value="B"), _rg("price", lt=0.2)])])]),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--top-k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--check", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from filter_expr_oracle import matches   # tests/ (the row-by-row evaluator)
    from sentio_b200 import payload_filter as pf
    from sentio_b200 import synth
    from sentio_b200.engine import B200Engine

    n, d, B, k = args.n_docs, args.dim, args.batch, args.top_k
    info = card()
    x16 = synth.dense_corpus(n, d)
    q = synth.query_vectors(B, d)
    rng = np.random.default_rng(2024)
    u = rng.random(n)
    bucket = np.full(n, 4, np.int32)
    for code, lo, hi in ((0, 0.0, 0.1), (1, 0.1, 0.11), (2, 0.11, 0.111), (3, 0.111, 0.1111)):
        bucket[(u >= lo) & (u < hi)] = code
    conds = {1.0: (0, 0), 0.1: (1, 0), 0.01: (1, 1), 0.001: (1, 2), 0.0001: (1, 3)}
    src, tag, year = rng.integers(0, 50, n), rng.integers(0, 10000, n), rng.integers(1990, 2026, n)
    price, tenant = rng.random(n), rng.integers(0, 4, n)
    payloads = [{"src": f"s{src[i]}", "tag": int(tag[i]), "year": int(year[i]), "price": float(price[i]),
                 "tenant": "ABCD"[tenant[i]]} for i in range(n)]

    eng = B200Engine(0)
    eng.load_dense(x16)
    eng.load_dense_tags(0, np.zeros(n, np.int32))
    eng.load_dense_tags(1, bucket)
    fb0 = eng.fallback_count()

    def timed(fn):
        t0 = time.perf_counter()
        fn()
        return time.perf_counter() - t0

    def mask_ms(fn, steps=5):
        eng.profile(True)
        for name in eng.PROF_IDS:
            eng.profile_read(name)
        for _ in range(steps):
            fn()
        out = {name + "_ms_per_call": round(eng.profile_read(name)[1] / steps, 4)
               for name in ("dense_filter_mask", "dense_scan", "dense_sample", "dense_filter_gather")}
        eng.profile(False)
        return out

    # (a) the fractions, legacy entry and programs alternated
    frac_rows = []
    for frac in FRACTIONS:
        f, c = conds[frac]
        legacy = (np.arange(B + 1, dtype=np.int32), np.full(B, f, np.int32), np.full(B, c, np.int32))
        prog = np.zeros(B, pf.PRED_DTYPE)
        prog["op"], prog["field"], prog["a"] = pf.EQ, f, c
        programs = (np.arange(B + 1, dtype=np.int32), prog, np.zeros(0, np.int32))
        run_l = lambda: eng.dense_topk(q, k, filters=legacy)            # noqa: E731
        run_p = lambda: eng.dense_topk_where(q, k, programs)            # noqa: E731
        for _ in range(args.warmup):
            run_l()
            run_p()
        tl, tp = [], []
        for _ in range(args.steps):
            tl.append(timed(run_l))
            tp.append(timed(run_p))
        a, b = run_l(), run_p()
        same = all(np.array_equal(x, y) for x, y in zip(a, b))
        frac_rows.append({"fraction": frac, "legacy_qps": round(B / float(np.median(tl)), 1),
                          "program_qps": round(B / float(np.median(tp)), 1),
                          "legacy": mask_ms(run_l), "program": mask_ms(run_p), "identical": bool(same)})

    # (b) shaped filters through programs
    idx = pf.PayloadIndex(payloads, lambda f, c: eng.load_dense_tags(f + 2, c), lambda *a: None,
                          lambda f, v: eng.load_dense_values(f, v), lambda *a: None)
    shaped = []
    for name, flt in SHAPED.items():
        off, prog, pool = idx.compile_programs([flt] * B)   # builds the columns the filter names
        tc = [timed(lambda: idx.compile_programs([flt] * B)) for _ in range(3)]
        prog["field"] = np.where(prog["op"] == pf.RANGE, prog["field"], np.where(prog["op"] <= pf.PRESENT,
                                                                                   prog["field"] + 2, prog["field"]))
        programs = (off, prog, pool)
        run = lambda: eng.dense_topk_where(q, k, programs)              # noqa: E731
        for _ in range(args.warmup):
            run()
        ts = [timed(run) for _ in range(args.steps)]
        prof = mask_ms(run)
        ids, sc, cnt = run()
        mask = np.fromiter((matches(flt, p) for p in payloads), bool, n)
        ok = True
        for b, (wi, ws) in enumerate(oracle_topk(x16, mask, q[:args.check], k)):
            ok &= int(cnt[b]) == len(wi) and np.array_equal(ids[b, :len(wi)], wi) and \
                np.allclose(sc[b, :len(wi)], ws, rtol=1e-9, atol=1e-12)
        shaped.append({"filter": name, "matching_rows": int(mask.sum()), "qps": round(B / float(np.median(ts)), 1),
                       "ms_median": round(float(np.median(ts)) * 1e3, 3),
                       "compile_ms_median": round(float(np.median(tc)) * 1e3, 3), **prof, "oracle_ok": bool(ok)})
    fb = eng.fallback_count() - fb0
    eng.close()
    line = json.dumps({"workload": f"{n}-doc synthetic, {d}-d, dense top_k={k}, {B}-query batches, host queries",
                       "card": info, "steps": args.steps, "warmup": args.warmup, "fallbacks": fb,
                       "fractions": frac_rows, "shaped": shaped})
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    ok = fb == 0 and all(r["oracle_ok"] for r in shaped) and all(r["identical"] for r in frac_rows)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
