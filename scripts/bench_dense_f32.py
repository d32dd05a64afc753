#!/usr/bin/env python
"""Float32 against float16 storage at bench scale (DESIGN.md K1g): the 1 M x 1024 synthetic directions of bench.py with
norms uniform in [0.5, 2] (as bench_dense_metric.py), loaded as a float16 and a float32 slot per metric (Cosine, Dot,
Euclid); 256-query device-resident batches, k = 100.

Steps of the two storages are alternated per metric in one process.  Per (metric, storage): queries/s, the fallbacks
per batch of the warmup and timed steps, the sampling / scan / select times per call (sb_profile, in separate profiled
steps after the timed ones) and, for float32, an fp64 check of a few queries against the vectors as given.  Then one
near-duplicate workload: a cluster of rows that store one fp16 row, queried near it (Cosine, both storages).  Reads the
card's name and power limit in the same run.  Prints one JSON line.

    python scripts/bench_dense_f32.py [--n-docs 1000000] [--dim 1024] [--steps 10] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

METRICS = ("cosine", "dot", "euclid")
STORAGES = ("float16", "float32")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the measurement stands; the card line says why it is missing
        return {"error": repr(e)}


def oracle_f32(x, q, k, metric, chunk=65536):
    """Exact fp64 top-k on the vectors as given: [(rows, scores) per query]."""
    q64 = q.astype(np.float64)
    best = [(np.zeros(0, np.int64), np.zeros(0)) for _ in range(len(q))]
    for lo in range(0, len(x), chunk):
        x64 = x[lo:lo + chunk].astype(np.float64)
        idx = lo + np.arange(len(x64))
        for b in range(len(q)):
            if metric == "euclid":
                t = q64[b][None, :] - x64
                s = np.sqrt((t * t).sum(1))
            elif metric == "dot":
                s = x64 @ q64[b]
            else:
                den = np.sqrt((x64 * x64).sum(1)) * np.sqrt(q64[b] @ q64[b])
                s = np.zeros(len(x64))
                np.divide(x64 @ q64[b], den, out=s, where=den > 0)
            bi = np.concatenate([best[b][0], idx])
            bs = np.concatenate([best[b][1], s])
            o = np.lexsort((bi, bs if metric == "euclid" else -bs))[:k]
            best[b] = (bi[o], bs[o])
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--top-k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--check", type=int, default=2, help="queries per metric checked against fp64 (float32 slots)")
    ap.add_argument("--dup", type=int, default=1000, help="rows of the near-duplicate cluster")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch

    from sentio_b200 import synth
    from sentio_b200.engine import B200Engine

    n, d, B, k = args.n_docs, args.dim, args.batch, args.top_k
    info = card()
    u = synth.dense_corpus(n, d)
    q = synth.query_vectors(B, d)
    rng = np.random.default_rng(7)
    x = np.empty((n, d), np.float32)
    nv = rng.uniform(0.5, 2.0, n)
    for lo in range(0, n, 65536):
        x[lo:lo + 65536] = u[lo:lo + 65536].astype(np.float32) * nv[lo:lo + 65536, None].astype(np.float32)
    del u
    dev = torch.device("cuda", 0)
    q_t = torch.from_numpy(q).to(dev)
    out = (torch.empty((B, k), dtype=torch.int64, device=dev), torch.empty((B, k), dtype=torch.float64, device=dev),
           torch.empty((B,), dtype=torch.int32, device=dev))

    def step(eng, qt):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.dense_topk_dev(qt, k, out=out)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def profile(eng, qt, steps=3):
        eng.profile(True)
        for name in eng.PROF_IDS:
            eng.profile_read(name)
        for _ in range(steps):
            step(eng, qt)
        prof = {}
        for name in ("dense_sample", "dense_scan", "dense_merge"):
            _, ms = eng.profile_read(name)
            prof[name + "_ms_per_call"] = round(ms / steps, 4)
        eng.profile(False)
        return prof

    def run_pair(engines, qt):
        """Alternate the storages step by step: {storage: (times, fallbacks of warmup + timed steps)}."""
        fb0 = {s: engines[s].fallback_count() for s in STORAGES}
        for _ in range(args.warmup):
            for s in STORAGES:
                step(engines[s], qt)
        times = {s: [] for s in STORAGES}
        for _ in range(args.steps):
            for s in STORAGES:
                times[s].append(step(engines[s], qt))
        return {s: (times[s], engines[s].fallback_count() - fb0[s]) for s in STORAGES}

    def row(t, fb):
        med = float(np.median(t))
        return {"qps": round(B / med, 1), "ms_median": round(med * 1e3, 3),
                "ms_min_max": [round(min(t) * 1e3, 3), round(max(t) * 1e3, 3)], "fallbacks": fb,
                "fallbacks_per_batch": round(fb / (args.steps + args.warmup), 2)}

    results = []
    for m in METRICS:
        engines = {s: B200Engine(0) for s in STORAGES}
        t_load = {}
        for s in STORAGES:
            t0 = time.perf_counter()
            engines[s].load_dense(x, metric=m, storage=s)
            t_load[s] = time.perf_counter() - t0
        runs = run_pair(engines, q_t)
        for s in STORAGES:
            prof = profile(engines[s], q_t)
            r = {"metric": m, "storage": s, **row(*runs[s]), **prof, "load_s": round(t_load[s], 2)}
            if s == "float32":
                ids, sc, cnt = (t.cpu().numpy() for t in out)
                ok = True
                for b, (wi, ws) in enumerate(oracle_f32(x, q[:args.check], k, m)):
                    ok &= int(cnt[b]) == len(wi) and np.array_equal(ids[b, :len(wi)], wi) and \
                        np.allclose(sc[b, :len(wi)], ws, rtol=1e-9, atol=1e-12 * max(1.0, float(np.abs(ws).max())))
                r["oracle_ok"] = bool(ok)
            results.append(r)
        for e in engines.values():
            e.close()

    # near-duplicates: --dup rows y0 + perturbations below a tenth of the fp16 spacing (one stored fp16 row), queries
    # near y0 so the whole cluster leads every ranking
    rng = np.random.default_rng(11)
    y0 = rng.standard_normal(d)
    y0 = (y0 / np.linalg.norm(y0)).astype(np.float16)
    sp = np.spacing(np.abs(y0)).astype(np.float64)
    start = n // 3
    x[start:start + args.dup] = (y0.astype(np.float64)[None, :] +
                                 rng.uniform(-0.1, 0.1, (args.dup, d)) * sp[None, :]).astype(np.float32)
    qd = (y0.astype(np.float32)[None, :] + 0.01 * rng.standard_normal((B, d))).astype(np.float32)
    qd_t = torch.from_numpy(qd).to(dev)
    engines = {s: B200Engine(0) for s in STORAGES}
    for s in STORAGES:
        engines[s].load_dense(x, storage=s)
    runs = run_pair(engines, qd_t)
    dup = []
    for s in STORAGES:
        prof = profile(engines[s], qd_t)
        ids = out[0].cpu().numpy()
        r = {"storage": s, **row(*runs[s]), **prof,
             "top_k_in_row_order": bool(all(ids[b].tolist() == list(range(start, start + k)) for b in range(B)))}
        if s == "float32":
            want = oracle_f32(x[start:start + args.dup], qd[:args.check], k, "cosine")
            r["oracle_ok"] = bool(all(np.array_equal(ids[b], start + wi) for b, (wi, _) in enumerate(want)))
        dup.append(r)
    for e in engines.values():
        e.close()

    line = json.dumps({"workload": f"{n}-doc synthetic directions, norms uniform in [0.5, 2], {d}-d, dense top_k={k}, "
                                   f"{B}-query batches, device-resident, float16 and float32 storage alternated per step",
                       "card": info, "steps": args.steps, "warmup": args.warmup, "results": results,
                       "near_duplicates": {"cluster_rows": args.dup, "metric": "cosine", "results": dup}})
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    ok = all(r.get("oracle_ok", True) for r in results + dup)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
