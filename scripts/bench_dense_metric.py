#!/usr/bin/env python
"""Dense search per distance metric at bench scale (DESIGN.md K1e): the 1 M x 1024 synthetic directions of bench.py,
given norms from three distributions (uniform in [0.5, 2], log-uniform over 1e-3 .. 1e3, uniform plus 10 outliers of
norm 1e4), loaded as Cosine, Dot and Euclid slots of the same directions; 256-query device-resident batches, k = 100.

Steps of the three metrics are alternated in one process.  Per (distribution, metric): queries/s, the sampling / scan /
select times per call (sb_profile, in separate profiled steps after the timed ones), the fallback count of the warmup
and timed steps, and an fp64 oracle check of a few queries.  The window size is not exposed by the library.  Prints
one JSON line.

    python scripts/bench_dense_metric.py [--n-docs 1000000] [--dim 1024] [--steps 10] [--warmup 2] [--out FILE]
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


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the measurement stands; the card line says why it is missing
        return {"error": repr(e)}


def norms(kind, n, rng):
    if kind == "uniform":
        return rng.uniform(0.5, 2.0, n)
    if kind == "loguniform":
        return 10.0 ** rng.uniform(-3.0, 3.0, n)
    v = rng.uniform(0.5, 2.0, n)
    v[rng.choice(n, 10, replace=False)] = 1e4
    return v


def oracle(x, q, k, metrics, chunk=65536):
    """Exact fp64 top-k per metric over the stored representation (y = fp16(x / ||x||), c = ||x|| / ||y||; cosine on y):
    {metric: [(rows, scores) per query]}."""
    q64 = q.astype(np.float64)
    res = {m: [(np.zeros(0, np.int64), np.zeros(0)) for _ in range(len(q))] for m in metrics}
    for lo in range(0, len(x), chunk):
        x64 = x[lo:lo + chunk].astype(np.float64)
        nrm = np.sqrt((x64 * x64).sum(1))
        y = (x64 / np.where(nrm > 0, nrm, 1.0)[:, None]).astype(np.float16).astype(np.float64)
        yn = np.sqrt((y * y).sum(1))
        c = np.zeros(len(y))
        np.divide(nrm, yn, out=c, where=yn > 0)
        idx = lo + np.arange(len(y))
        for metric, b in [(m, b) for m in metrics for b in range(len(q))]:
            best = res[metric]
            if metric == "cosine":
                s = np.zeros(len(y))
                np.divide(y @ q64[b], yn * np.sqrt(q64[b] @ q64[b]), out=s, where=yn > 0)
                key = -s
            elif metric == "dot":
                s = c * (y @ q64[b])
                key = -s
            else:
                diff = q64[b][None, :] - c[:, None] * y
                s = np.sqrt((diff * diff).sum(1))
                key = s
            bi = np.concatenate([best[b][0], idx])
            bs = np.concatenate([best[b][1], s])
            bk = np.concatenate([(-best[b][1] if metric != "euclid" else best[b][1]), key])
            o = np.lexsort((bi, bk))[:k]
            best[b] = (bi[o], bs[o])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--top-k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dists", default="uniform,loguniform,outliers")
    ap.add_argument("--check", type=int, default=2, help="queries per (distribution, metric) checked against fp64")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch

    from sentio_b200 import synth
    from sentio_b200.engine import B200Engine

    n, d, B, k = args.n_docs, args.dim, args.batch, args.top_k
    info = card()
    u = synth.dense_corpus(n, d)
    q = synth.query_vectors(B, d)
    dev = torch.device("cuda", 0)
    q_t = torch.from_numpy(q).to(dev)
    engines = {m: B200Engine(0) for m in METRICS}
    outs = {m: (torch.empty((B, k), dtype=torch.int64, device=dev), torch.empty((B, k), dtype=torch.float64, device=dev),
                torch.empty((B,), dtype=torch.int32, device=dev)) for m in METRICS}

    def step(m):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        engines[m].dense_topk_dev(q_t, k, out=outs[m])
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    results = []
    for dist in args.dists.split(","):
        rng = np.random.default_rng(7)
        x = np.empty((n, d), np.float32)
        nv = norms(dist, n, rng)
        for lo in range(0, n, 65536):
            x[lo:lo + 65536] = u[lo:lo + 65536].astype(np.float32) * nv[lo:lo + 65536, None].astype(np.float32)
        t_load = {}
        for m in METRICS:
            t0 = time.perf_counter()
            engines[m].load_dense(x, metric=m)
            t_load[m] = time.perf_counter() - t0
        fb0 = {m: engines[m].fallback_count() for m in METRICS}
        for _ in range(args.warmup):
            for m in METRICS:
                step(m)
        times = {m: [] for m in METRICS}
        for _ in range(args.steps):
            for m in METRICS:
                times[m].append(step(m))
        fb_run = {m: engines[m].fallback_count() - fb0[m] for m in METRICS}   # warmup + timed steps
        prof_steps = 3
        want = oracle(x, q[:args.check], k, METRICS)
        for m in METRICS:
            eng = engines[m]
            eng.profile(True)
            for name in eng.PROF_IDS:
                eng.profile_read(name)
            for _ in range(prof_steps):
                step(m)
            prof = {}
            for name in ("dense_sample", "dense_scan", "dense_merge"):
                _, ms = eng.profile_read(name)
                prof[name + "_ms_per_call"] = round(ms / prof_steps, 4)
            eng.profile(False)
            ids, sc, cnt = (t.cpu().numpy() for t in outs[m])
            ok = True
            for b, (wi, ws) in enumerate(want[m]):
                ok &= int(cnt[b]) == len(wi) and np.array_equal(ids[b, :len(wi)], wi) and \
                    np.allclose(sc[b, :len(wi)], ws, rtol=1e-9, atol=1e-12 * max(1.0, float(np.abs(ws).max())))
            t = times[m]
            med = float(np.median(t))
            results.append({"norms": dist, "metric": m, "qps": round(B / med, 1), "ms_median": round(med * 1e3, 3),
                            "ms_min_max": [round(min(t) * 1e3, 3), round(max(t) * 1e3, 3)],
                            "fallbacks": fb_run[m], "fallbacks_per_batch": round(fb_run[m] / (args.steps + args.warmup), 2),
                            **prof, "load_s": round(t_load[m], 2), "oracle_ok": bool(ok)})
        del x
    for e in engines.values():
        e.close()
    line = json.dumps({"workload": f"{n}-doc synthetic directions, {d}-d, dense top_k={k}, {B}-query batches, "
                                   "device-resident, metrics alternated per step",
                       "card": info, "steps": args.steps, "warmup": args.warmup,
                       "window_size": "not exposed by the library", "results": results})
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    return 0 if all(r["oracle_ok"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
