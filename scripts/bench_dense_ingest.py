#!/usr/bin/env python
"""Dense slot mutation at bench scale: a 1 M x 1024 collection (the synthetic corpus of bench.py).

Measures, with a host clock around each call (every mutating call returns after its device work is done):
  * upsert rows/s for batches of 1, 256, 4096 and 65 536 fp32 rows, as appends and as overwrites of random rows, from
    pageable and from page-locked (sb_host_alloc) input;
  * delete rows/s for batches of 1, 256 and 4096 random rows;
  * the time of a growth reallocation (an append that outgrows the capacity, minus the same append within
    capacity), 5 repetitions on a freshly loaded slot each;
  * unfiltered 256-query q/s (k = 100, device-resident queries) on the collection after >= 100 k row mutations,
    alternated with a fresh load of the same rows, whose outputs must be bit-identical.
Prints one JSON line (and writes it to --out).

    python scripts/bench_dense_ingest.py [--n-docs 1000000] [--dim 1024] [--steps 20] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

UPSERT_BATCHES = {1: 200, 256: 40, 4096: 10, 65536: 3}   # batch -> timed calls
DELETE_BATCHES = {1: 200, 256: 40, 4096: 10}
GROWTH_REPS = 5


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the measurement stands; the card line says why it is missing
        return {"error": repr(e)}


def timed(fn):
    t = time.perf_counter()
    fn()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from sentio_b200 import synth
    from sentio_b200.engine import B200Engine

    n, d = args.n_docs, args.dim
    rng = np.random.default_rng(0)
    x16 = synth.dense_corpus(n, d)
    eng = B200Engine(0)
    res = {"metric": "dense_ingest", "n_docs": n, "dim": d, "card": card()}

    # ---- growth reallocation, GROWTH_REPS times: each load gives capacity round_up(n, 128); an append past it
    # reallocates to 1.5 x.  Realloc time = that append minus the same append within capacity, on the same slot.
    cap = (n + 127) // 128 * 128
    m = cap - n + 1
    grow_vecs = rng.standard_normal((m, d)).astype(np.float32)
    t_grow, t_plain = [], []
    for _ in range(GROWTH_REPS):
        eng.load_dense(x16)
        t_grow.append(timed(lambda: eng.dense_upsert(np.arange(n, n + m), grow_vecs)))
        eng.dense_delete(np.arange(n, n + m))
        t_plain.append(timed(lambda: eng.dense_upsert(np.arange(n, n + m), grow_vecs)))
        eng.dense_delete(np.arange(n, n + m))
    realloc = [1e3 * (a - b) for a, b in zip(t_grow, t_plain)]
    res["growth"] = {"from_rows": cap, "to_rows": (cap + cap // 2 + 127) // 128 * 128, "append_rows": m,
                     "reps": GROWTH_REPS, "append_with_growth_ms": [1e3 * t for t in t_grow],
                     "append_within_capacity_ms": [1e3 * t for t in t_plain], "realloc_ms": realloc,
                     "realloc_ms_median": float(np.median(realloc))}
    print(json.dumps(res["growth"]), file=sys.stderr)

    # ---- upserts: append and overwrite, pageable and page-locked input
    eng.dense_reserve(n + sum(b * r for b, r in UPSERT_BATCHES.items()) + 1024)
    up = []
    for batch, reps in UPSERT_BATCHES.items():
        src = rng.standard_normal((batch, d)).astype(np.float32)
        pinned = eng.pinned_empty((batch, d), np.float32)
        pinned[:] = src
        for kind, vecs in (("pageable", src), ("page_locked", pinned)):
            eng.dense_upsert(rng.choice(n, batch, replace=False), vecs)   # warm-up (staging buffers)
            rows = [rng.choice(n, batch, replace=False) for _ in range(reps)]
            t_over = sum(timed(lambda r=r: eng.dense_upsert(r, vecs)) for r in rows)
            cur = eng.dense_count[0]
            t_app = 0.0
            for i in range(reps):
                r = np.arange(cur + i * batch, cur + (i + 1) * batch)
                t_app += timed(lambda r=r: eng.dense_upsert(r, vecs))
            eng.dense_delete(np.arange(cur, eng.dense_count[0]))           # back to n rows (tail only: no moves)
            up.append({"batch": batch, "input": kind, "calls": reps,
                       "overwrite_rows_per_s": batch * reps / t_over, "overwrite_ms_per_call": 1e3 * t_over / reps,
                       "append_rows_per_s": batch * reps / t_app, "append_ms_per_call": 1e3 * t_app / reps})
            print(json.dumps(up[-1]), file=sys.stderr)
    res["upsert"] = up

    # ---- deletes of random rows (moves from the tail); the collection is not refilled, so it shrinks by the total
    dl = []
    for batch, reps in DELETE_BATCHES.items():
        t = 0.0
        for _ in range(reps):
            rows = rng.choice(eng.dense_count[0], batch, replace=False)
            t += timed(lambda r=rows: eng.dense_delete(r))
        dl.append({"batch": batch, "calls": reps, "rows_per_s": batch * reps / t, "ms_per_call": 1e3 * t / reps})
        print(json.dumps(dl[-1]), file=sys.stderr)
    res["delete"] = dl

    # ---- >= 100 k mutations in 4096-row batches (overwrites, deletes, appends), then search vs a fresh load
    mutated = 0
    while mutated < 100_000:
        c = eng.dense_count[0]
        eng.dense_upsert(rng.choice(c, 4096, replace=False), rng.standard_normal((4096, d)).astype(np.float32))
        eng.dense_delete(rng.choice(c, 4096, replace=False))
        c = eng.dense_count[0]
        eng.dense_upsert(np.arange(c, c + 4096), rng.standard_normal((4096, d)).astype(np.float32))
        mutated += 3 * 4096
    c = eng.dense_count[0]
    rows16 = np.empty((c, d), np.float16)
    for lo in range(0, c, 65536):
        rows16[lo:lo + 65536] = eng.dense_fetch(np.arange(lo, min(c, lo + 65536))).astype(np.float16)
    fresh = B200Engine(0)
    fresh.load_dense(rows16)
    del rows16
    q = torch.from_numpy(synth.query_vectors(256, d)).cuda()
    k = 100
    outs = {}
    for name, e in (("mutated", eng), ("fresh", fresh)):
        for _ in range(3):
            outs[name] = [t.cpu() for t in e.dense_topk_dev(q, k)]
    torch.cuda.synchronize()
    identical = all(torch.equal(a, b) for a, b in zip(outs["mutated"], outs["fresh"]))
    times = {"mutated": [], "fresh": []}
    for _ in range(args.steps):
        for name, e in (("mutated", eng), ("fresh", fresh)):
            torch.cuda.synchronize()
            t = time.perf_counter()
            e.dense_topk_dev(q, k)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t)
    res["search_after_mutations"] = {
        "rows_mutated": mutated, "rows": c, "batch": 256, "k": k, "steps": args.steps, "bit_identical": identical,
        "mutated_qps_median": 256 / float(np.median(times["mutated"])),
        "fresh_qps_median": 256 / float(np.median(times["fresh"])),
        "fallbacks": [eng.fallback_count(), fresh.fallback_count()]}
    fresh.close()
    eng.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not identical:
        sys.exit("search after mutations differs from a fresh load")


if __name__ == "__main__":
    main()
