#!/usr/bin/env python
"""Uint8 against float16 storage of the same integer rows (DESIGN.md K1i): 1 M x 1024, once uniform bytes and once the
quantised clustered corpus round(128 + 40 g) clipped to [0, 255]; Cosine, Dot and Euclid; device-resident batches of
16, 64, 128 and 256 queries, k = 100.

Per (corpus, metric, batch) the two slots are alternated step by step after warmup steps.  Per slot: queries/s, the
sampling / scan / select times per call (sb_profile, in separate profiled steps after the timed ones), fallbacks per
batch, the HBM bytes one full scan pass reads (computed from shapes: rows + per-row scales) and the GB/s that gives over
the profiled scan time.  The uint8 slot's answers to 8 queries are checked against an fp64 oracle on x.  Reads the
card's name and power limit in the same run.  Prints one JSON line.

    python scripts/bench_dense_u8.py [--n-docs 1000000] [--dim 1024] [--steps 10] [--warmup 3] [--out FILE]
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
STORAGES = ("float16", "uint8")
BATCHES = (16, 64, 128, 256)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the measurement stands; the card line says why it is missing
        return {"error": repr(e)}


def make_corpus(kind, n, d, seed=5):
    rng = np.random.default_rng(seed)
    x = np.empty((n, d), np.uint8)
    c = rng.standard_normal((64, d)).astype(np.float32)
    for lo in range(0, n, 65536):
        m = min(65536, n - lo)
        if kind == "uniform":
            x[lo:lo + m] = rng.integers(0, 256, (m, d), dtype=np.uint8)
        else:
            g = c[rng.integers(0, 64, m)] * 0.5 + rng.standard_normal((m, d), dtype=np.float32)
            x[lo:lo + m] = np.clip(np.rint(128 + 40 * g), 0, 255)
    return x


def oracle(x_t, q, k, metric, chunk=65536):
    """Exact fp64 top-k on the integer rows (x_t: the uint8 rows on the device; fp64 arithmetic by torch, chunked):
    [(rows, scores) per query]."""
    import torch

    q64 = torch.from_numpy(q.astype(np.float64)).to(x_t.device)
    best = [(np.zeros(0, np.int64), np.zeros(0)) for _ in range(len(q))]
    for lo in range(0, x_t.shape[0], chunk):
        x64 = x_t[lo:lo + chunk].double()
        idx = lo + np.arange(x64.shape[0])
        for b in range(len(q)):
            if metric == "euclid":
                s = torch.sqrt(((q64[b][None, :] - x64) ** 2).sum(1))
            elif metric == "dot":
                s = x64 @ q64[b]
            else:
                den = torch.sqrt((x64 * x64).sum(1)) * torch.sqrt(q64[b] @ q64[b])
                s = torch.where(den > 0, (x64 @ q64[b]) / torch.where(den > 0, den, 1.0), 0.0)
            s = s.cpu().numpy()
            bi = np.concatenate([best[b][0], idx])
            bs = np.concatenate([best[b][1], s])
            o = np.lexsort((bi, bs if metric == "euclid" else -bs))[:k]
            best[b] = (bi[o], bs[o])
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--top-k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", type=int, default=8, help="queries per (corpus, metric) checked against fp64")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch

    from sentio_b200.engine import B200Engine

    n, d, k = args.n_docs, args.dim, args.top_k
    info = card()
    n_pad = (n + 127) // 128 * 128
    d_pad = {"float16": (d + 7) // 8 * 8, "uint8": (d + 63) // 64 * 64}
    # bytes one full scan pass reads: the rows and the per-row scale (Euclid: + h)
    pass_bytes = {(s, m): n_pad * d_pad[s] * (2 if s == "float16" else 1) + n_pad * (8 if m == "euclid" else 4)
                  for s in STORAGES for m in METRICS}
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(9)

    def step(eng, qt, out):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.dense_topk_dev(qt, k, out=out)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def profile(eng, qt, out, steps=3):
        eng.profile(True)
        for name in eng.PROF_IDS:
            eng.profile_read(name)
        for _ in range(steps):
            step(eng, qt, out)
        prof = {}
        for name in ("dense_sample", "dense_scan", "dense_merge"):
            _, ms = eng.profile_read(name)
            prof[name + "_ms_per_call"] = round(ms / steps, 4)
        eng.profile(False)
        return prof

    results = []
    t_start = time.perf_counter()

    def progress(*a):   # one line per step of the run, so a long run shows where it is
        print(f"[{time.perf_counter() - t_start:7.1f} s]", *a, file=sys.stderr, flush=True)

    for kind in ("uniform", "clustered"):
        x = make_corpus(kind, n, d)
        x_t = torch.from_numpy(x).to(dev)
        progress("corpus", kind)
        q_all = (rng.standard_normal((max(BATCHES), d)) * 40 + 128).astype(np.float32)
        for m in METRICS:
            engines = {s: B200Engine(0) for s in STORAGES}
            t_load = {}
            for s in STORAGES:
                t0 = time.perf_counter()
                engines[s].load_dense(x if s == "uint8" else x.astype(np.float16), metric=m, storage=s)
                t_load[s] = round(time.perf_counter() - t0, 2)
                progress("loaded", kind, m, s, t_load[s], "s")
            for B in BATCHES:
                qt = torch.from_numpy(q_all[:B]).to(dev)
                outs = {s: (torch.empty((B, k), dtype=torch.int64, device=dev),
                            torch.empty((B, k), dtype=torch.float64, device=dev),
                            torch.empty((B,), dtype=torch.int32, device=dev)) for s in STORAGES}
                fb0 = {s: engines[s].fallback_count() for s in STORAGES}
                for _ in range(args.warmup):
                    for s in STORAGES:
                        step(engines[s], qt, outs[s])
                times = {s: [] for s in STORAGES}
                for _ in range(args.steps):
                    for s in STORAGES:
                        times[s].append(step(engines[s], qt, outs[s]))
                for s in STORAGES:
                    fb = engines[s].fallback_count() - fb0[s]
                    prof = profile(engines[s], qt, outs[s])
                    med = float(np.median(times[s]))
                    scan_ms = prof["dense_scan_ms_per_call"]
                    r = {"corpus": kind, "metric": m, "batch": B, "storage": s, "qps": round(B / med, 1),
                         "ms_median": round(med * 1e3, 3),
                         "ms_min_max": [round(min(times[s]) * 1e3, 3), round(max(times[s]) * 1e3, 3)],
                         "fallbacks_per_batch": round(fb / (args.steps + args.warmup), 2), **prof,
                         "scan_pass_bytes": pass_bytes[(s, m)],
                         "scan_gb_per_s": round(pass_bytes[(s, m)] / (scan_ms * 1e-3) / 1e9, 1) if scan_ms > 0 else None,
                         "load_s": t_load[s]}
                    if s == "uint8" and B == BATCHES[-1]:
                        ids, sc, cnt = (t.cpu().numpy() for t in outs[s])
                        ok = True
                        for b, (wi, ws) in enumerate(oracle(x_t, q_all[:args.check], k, m)):
                            ok &= int(cnt[b]) == len(wi) and np.array_equal(ids[b, :len(wi)], wi) and \
                                np.allclose(sc[b, :len(wi)], ws, rtol=1e-9, atol=1e-12 * max(1.0, float(np.abs(ws).max())))
                        r["oracle_ok"] = bool(ok)
                    results.append(r)
                    progress(json.dumps(r))
            for e in engines.values():
                e.close()
        del x, x_t

    line = json.dumps({"workload": f"{n} x {d} uint8 rows (uniform bytes / quantised clustered), dense top_k={k}, "
                                   f"device-resident batches {list(BATCHES)}, float16 and uint8 slots of the same rows "
                                   "alternated per step",
                       "card": info, "steps": args.steps, "warmup": args.warmup, "results": results})
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    return 0 if all(r.get("oracle_ok", True) for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
