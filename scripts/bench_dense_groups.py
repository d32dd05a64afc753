#!/usr/bin/env python
"""Grouped dense search at bench scale (DESIGN.md K1f): the 1 M x 1024 synthetic Cosine corpus of bench.py with a group
key of ~20 rows per group ("uniform": row // 20 of a random permutation) and a skewed variant (a few groups of tens of
thousands of rows, a long tail of small ones); 256-query batches from host memory, (limit, group_size) = (10, 3).

Grouped steps and plain top-100 steps of the same queries alternate in one process.  Per key: queries/s of both, the
per-stage device times of the grouped call (sb_profile, in separate profiled steps after the timed ones), the histogram
of rounds per query, the fallback count, and an fp64 oracle check of 8 queries.  Prints one JSON line.

    python scripts/bench_dense_groups.py [--n-docs 1000000] [--dim 1024] [--steps 10] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_dense_metric import card  # noqa: E402
from groups_oracle import group_search  # noqa: E402

STAGES = ("dense_sample", "dense_scan", "dense_merge", "dense_filter_mask", "dense_filter_gather", "dense_group_collect",
          "dense_group_assemble")


def cosine_scores(u, q, chunk=16384):
    """fp64 cosine of every stored row (fp16 rows as loaded from fp16 input) against each query: [len(q), n]."""
    q64 = q.astype(np.float64)
    q64 /= np.linalg.norm(q64, axis=1, keepdims=True)
    out = np.empty((len(q), len(u)))
    for lo in range(0, len(u), chunk):
        y = u[lo:lo + chunk].astype(np.float64)
        yn = np.sqrt((y * y).sum(1))
        s = np.zeros((len(y), len(q)))
        np.divide(y @ q64.T, yn[:, None], out=s, where=yn[:, None] > 0)
        out[:, lo:lo + chunk] = s.T
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--limit", type=int, default=10)
    ap.add_argument("--group-size", type=int, default=3)
    ap.add_argument("--top-k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--check", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from sentio_b200 import synth
    from sentio_b200.engine import B200Engine

    n, d, B, L, G, k = args.n_docs, args.dim, args.batch, args.limit, args.group_size, args.top_k
    info = card()
    u = synth.dense_corpus(n, d)
    q = synth.query_vectors(B, d)
    rng = np.random.default_rng(11)
    keys = {"uniform": (rng.permutation(n) // 20).astype(np.int32),
            "skewed": np.floor((n // 20) * rng.random(n) ** 4).astype(np.int32)}
    eng = B200Engine(0)
    eng.load_dense(u)
    exact = cosine_scores(u, q[:args.check])
    results = []
    for name, codes in keys.items():
        eng.load_dense_tags(0, codes)
        sizes = np.bincount(codes)
        fb0 = eng.fallback_count()
        r0 = eng.dense_group_rounds(8)
        tg, tp = [], []
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            got = eng.dense_groups(q, 0, L, G)
            t1 = time.perf_counter()
            eng.dense_topk(q, k)
            t2 = time.perf_counter()
            if i >= args.warmup:
                tg.append(t1 - t0)
                tp.append(t2 - t1)
        fb = eng.fallback_count() - fb0
        rounds = (eng.dense_group_rounds(8) - r0).tolist()
        eng.profile(True)
        for s in eng.PROF_IDS:
            eng.profile_read(s)
        prof_steps = 3
        for _ in range(prof_steps):
            eng.dense_groups(q, 0, L, G)
        prof = {}
        for s in STAGES:
            cnt, ms = eng.profile_read(s)
            prof[s] = {"launches_per_call": round(cnt / prof_steps, 2), "ms_per_call": round(ms / prof_steps, 4)}
        eng.profile(False)
        ng, gc, gh, ids, sc = got
        ok = True
        groups = codes.tolist()
        for b in range(args.check):
            want = group_search(exact[b], groups, L, G)
            ok &= int(ng[b]) == len(want)
            for g, (code, rows) in enumerate(want):
                ok &= int(gc[b, g]) == code and int(gh[b, g]) == len(rows)
                ok &= list(map(int, ids[b, g, :len(rows)])) == [r for r, _ in rows]
                ok &= bool(np.allclose(sc[b, g, :len(rows)], [s for _, s in rows], rtol=1e-9, atol=1e-12))
        mg, mp = float(np.median(tg)), float(np.median(tp))
        results.append({"key": name, "groups": int((sizes > 0).sum()), "largest_group": int(sizes.max()),
                        "groups_qps": round(B / mg, 1), "groups_ms_median": round(mg * 1e3, 3),
                        "groups_ms_min_max": [round(min(tg) * 1e3, 3), round(max(tg) * 1e3, 3)],
                        "topk_qps": round(B / mp, 1), "topk_ms_median": round(mp * 1e3, 3),
                        "rounds_hist": rounds, "fallbacks": fb, "stages": prof, "oracle_ok": bool(ok)})
    eng.close()
    line = json.dumps({"workload": f"{n}-doc synthetic directions, {d}-d, Cosine, search_groups limit={L} "
                                   f"group_size={G} vs top_k={k}, {B}-query host batches, alternated per step",
                       "card": info, "steps": args.steps, "warmup": args.warmup,
                       "rounds_hist": "[r] = queries answered in r + 1 rounds, warmup and timed steps",
                       "results": results})
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    return 0 if all(r["oracle_ok"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
