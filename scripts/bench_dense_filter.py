#!/usr/bin/env python
"""Filtered dense search at bench scale: 1 M x 1024 synthetic corpus (the seeds of bench.py), 256-query batches of
device-resident queries, k = 100, a payload field whose values match 100 %, 10 %, 1 %, 0.1 % and 0.01 % of the rows.

Each filtered step is alternated with an unfiltered step in the same process.  Per fraction: queries/s of both, the
mask-build, scan and gather-path times per call (sb_profile, CUDA events, in separate profiled steps after the timed
ones), an oracle check of 8 queries, and the fallback counter (which must not move).  Prints one JSON line.

    python scripts/bench_dense_filter.py [--n-docs 1000000] [--dim 1024] [--steps 20] [--warmup 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FRACTIONS = [1.0, 0.1, 0.01, 0.001, 0.0001]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the measurement stands; the card line says why it is missing
        return {"error": repr(e)}


def oracle_topk(x16, mask, q, k, chunk=65536):
    """Exact (score desc, row asc) top-k of the rows where mask is set, fp64, chunked over the corpus."""
    q64 = q.astype(np.float64)
    qn = np.sqrt((q64 * q64).sum(1))
    best = [(np.zeros(0, np.int64), np.zeros(0)) for _ in range(len(q))]
    for lo in range(0, len(x16), chunk):
        idx = lo + np.flatnonzero(mask[lo:lo + chunk])
        if len(idx) == 0:
            continue
        x = x16[idx].astype(np.float64)
        xn = np.sqrt((x * x).sum(1))
        dots = x @ q64.T
        for b in range(len(q)):
            den = xn * qn[b]
            s = np.zeros(len(x))
            np.divide(dots[:, b], den, out=s, where=den > 0)
            bi = np.concatenate([best[b][0], idx])
            bs = np.concatenate([best[b][1], s])
            o = np.lexsort((bi, -bs))[:k]
            best[b] = (bi[o], bs[o])
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--top-k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", type=int, default=8, help="queries per fraction checked against the fp64 oracle")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch

    from sentio_b200 import synth
    from sentio_b200.engine import B200Engine

    n, d, B, k = args.n_docs, args.dim, args.batch, args.top_k
    info = card()
    x16 = synth.dense_corpus(n, d)
    q = synth.query_vectors(B, d)
    rng = np.random.default_rng(2024)
    # field 0: every row has the same value (100 %); field 1: disjoint buckets of 10 %, 1 %, 0.1 %, 0.01 % (+ the rest)
    u = rng.random(n)
    bucket = np.full(n, 4, np.int32)
    for code, lo, hi in ((0, 0.0, 0.1), (1, 0.1, 0.11), (2, 0.11, 0.111), (3, 0.111, 0.1111)):
        bucket[(u >= lo) & (u < hi)] = code
    conds = {1.0: (0, 0), 0.1: (1, 0), 0.01: (1, 1), 0.001: (1, 2), 0.0001: (1, 3)}

    eng = B200Engine(0)
    eng.load_dense(x16)
    eng.load_dense_tags(0, np.zeros(n, np.int32))
    eng.load_dense_tags(1, bucket)
    dev = torch.device("cuda", 0)
    q_t = torch.from_numpy(q).to(dev)
    out = (torch.empty((B, k), dtype=torch.int64, device=dev), torch.empty((B, k), dtype=torch.float64, device=dev),
           torch.empty((B,), dtype=torch.int32, device=dev))
    fb0 = eng.fallback_count()

    def step(filters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.dense_topk_dev(q_t, k, out=out, filters=filters)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    results = []
    for frac in FRACTIONS:
        f, c = conds[frac]
        flt = tuple(torch.from_numpy(a).to(dev) for a in (np.arange(B + 1, dtype=np.int32), np.full(B, f, np.int32),
                                                            np.full(B, c, np.int32)))
        matching = int(np.count_nonzero((bucket if f == 1 else np.zeros(n, np.int32)) == c))
        for _ in range(args.warmup):
            step(flt)
            step(None)
        tf, tu = [], []
        for _ in range(args.steps):
            tf.append(step(flt))
            tu.append(step(None))
        # kernel breakdown in separate, profiled steps
        eng.profile(True)
        for name in eng.PROF_IDS:
            eng.profile_read(name)
        prof_steps = 5
        for _ in range(prof_steps):
            step(flt)
        prof = {}
        for name in ("dense_filter_mask", "dense_sample", "dense_scan", "dense_merge", "dense_filter_gather"):
            cnt, ms = eng.profile_read(name)
            prof[name + "_ms_per_call"] = round(ms / prof_steps, 4)
        eng.profile(False)
        # oracle check of the last batch's first queries
        eng.dense_topk_dev(q_t, k, out=out, filters=flt)
        torch.cuda.synchronize()
        ids, sc, cnt = (t.cpu().numpy() for t in out)
        mask = (bucket == c) if f == 1 else np.ones(n, bool)
        ok = True
        for b, (wi, ws) in enumerate(oracle_topk(x16, mask, q[:args.check], k)):
            ok &= int(cnt[b]) == len(wi) and np.array_equal(ids[b, :len(wi)], wi) and \
                np.allclose(sc[b, :len(wi)], ws, rtol=1e-9, atol=1e-12)
        med_f, med_u = float(np.median(tf)), float(np.median(tu))
        results.append({"fraction": frac, "matching_rows": matching,
                        "filtered_qps": round(B / med_f, 1), "unfiltered_qps": round(B / med_u, 1),
                        "filtered_ms_median": round(med_f * 1e3, 3), "unfiltered_ms_median": round(med_u * 1e3, 3),
                        "filtered_ms_min_max": [round(min(tf) * 1e3, 3), round(max(tf) * 1e3, 3)],
                        **prof, "oracle_ok": bool(ok)})
    fb = eng.fallback_count() - fb0
    eng.close()
    line = json.dumps({"workload": f"{n}-doc synthetic, {d}-d, dense top_k={k}, {B}-query batches, device-resident",
                       "card": info, "steps": args.steps, "warmup": args.warmup, "fallbacks": fb,
                       "results": results})
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    return 0 if fb == 0 and all(r["oracle_ok"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
