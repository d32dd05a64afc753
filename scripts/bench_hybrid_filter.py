#!/usr/bin/env python
"""Filtered hybrid retrieval at bench scale: the 1 M x 1024 dense corpus and the 1 M-doc Zipf BM25 corpus of bench.py
(same seeds), 128-query rrf batches from host buffers (``hybrid_topk``, the sb_hybrid_topk[_filtered] entry point),
k = 100, one payload field whose values match 100 %, 10 %, 1 %, 0.1 % and 0.01 % of the docs, the same codes loaded for
dense slot 0 and for BM25.

Each filtered step is alternated with an unfiltered step in the same process.  Per fraction: queries/s of both, the
per-stage device times per call from sb_profile (BM25 score and select; dense mask, gather, sample, scan and merge) in
separate profiled steps after the timed ones, and a check of a few queries against oracle.fusion over the filtered
dense oracle and FastBM25 masked by the filter.  Prints one JSON line.

    python scripts/bench_hybrid_filter.py [--n-docs 1000000] [--dim 1024] [--steps 20] [--warmup 3] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_dense_filter import card, oracle_topk  # noqa: E402

FRACTIONS = [1.0, 0.1, 0.01, 0.001, 0.0001]
STAGES = ("bm25_score", "bm25_select", "dense_filter_mask", "dense_filter_gather", "dense_sample", "dense_scan",
          "dense_merge", "fuse")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--top-k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check", type=int, default=4, help="queries per fraction checked against the oracles")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import bm25_filter_oracle as fo
    from oracle import fusion as fusion_oracle
    from oracle.rank_bm25_port import FastBM25
    from sentio_b200 import synth
    from sentio_b200.engine import B200Engine
    from sentio_b200.index import build_bm25_from_token_ids

    n, d, B, k = args.n_docs, args.dim, args.batch, args.top_k
    info = card()
    x16 = synth.dense_corpus(n, d)
    q = synth.query_vectors(B, d)
    flat, off = synth.text_corpus_tokens(n)
    idx = build_bm25_from_token_ids(flat, off)
    terms = [idx.term_ids(t) for t in synth.query_tokens(B)]
    rng = np.random.default_rng(2024)
    # field 0: every doc has the same value (100 %); field 1: disjoint buckets of 10 %, 1 %, 0.1 %, 0.01 % (+ the rest)
    u = rng.random(n)
    bucket = np.full(n, 4, np.int32)
    for code, lo, hi in ((0, 0.0, 0.1), (1, 0.1, 0.11), (2, 0.11, 0.111), (3, 0.111, 0.1111)):
        bucket[(u >= lo) & (u < hi)] = code
    conds = {1.0: (0, 0), 0.1: (1, 0), 0.01: (1, 1), 0.001: (1, 2), 0.0001: (1, 3)}

    eng = B200Engine(0)
    eng.load_dense(x16)
    eng.load_bm25(idx)
    for f, col in ((0, np.zeros(n, np.int32)), (1, bucket)):
        eng.load_dense_tags(f, col)
        eng.load_bm25_tags(f, col)
    qf, qo = eng.pack_queries(terms)
    fast = FastBM25(idx.indptr, idx.post_doc, idx.post_tf, idx.doc_len, idx.idf, idx.avgdl, idx.variant, idx.k1,
                    idx.b, idx.delta)

    def step(filters):
        t0 = time.perf_counter()
        r = eng.hybrid_topk(q, qf, qo, k, "rrf", 60, 0.5, 0.5, filters=filters)   # returns after its own D2H
        return time.perf_counter() - t0, r

    results = []
    for frac in FRACTIONS:
        f, c = conds[frac]
        flt = (np.arange(B + 1, dtype=np.int32), np.full(B, f, np.int32), np.full(B, c, np.int32))
        mask = (bucket == c) if f == 1 else np.ones(n, bool)
        for _ in range(args.warmup):
            step(flt)
            step(None)
        tf, tu = [], []
        for _ in range(args.steps):
            tf.append(step(flt)[0])
            tu.append(step(None)[0])
        # per-stage device times in separate, profiled steps
        eng.profile(True)
        for name in eng.PROF_IDS:
            eng.profile_read(name)
        prof_steps = 5
        for _ in range(prof_steps):
            step(flt)
        prof = {}
        for name in STAGES:
            _, ms = eng.profile_read(name)
            prof[name + "_ms_per_call"] = round(ms / prof_steps, 4)
        eng.profile(False)
        # oracle check of the first queries
        _, (ids, sc, _src, cnt) = step(flt)
        ok = True
        for b, (di, ds) in enumerate(oracle_topk(x16, mask, q[:args.check], k)):
            s = fast.get_scores(list(terms[b]))
            sl = [(int(i), float(s[i])) for i in fo.filtered_topk(s, mask, k)]
            want = fusion_oracle.fuse("rrf", 60, 0.5, 0.5, list(zip(di.tolist(), ds.tolist())), sl, [], k)
            m = int(cnt[b])
            ok &= m == len(want) and ids[b, :m].tolist() == [w[0] for w in want] and \
                sc[b, :m].tolist() == [w[1] for w in want]
        med_f, med_u = float(np.median(tf)), float(np.median(tu))
        results.append({"fraction": frac, "matching_docs": int(np.count_nonzero(mask)),
                        "filtered_qps": round(B / med_f, 1), "unfiltered_qps": round(B / med_u, 1),
                        "filtered_ms_median": round(med_f * 1e3, 3), "unfiltered_ms_median": round(med_u * 1e3, 3),
                        "filtered_ms_min_max": [round(min(tf) * 1e3, 3), round(max(tf) * 1e3, 3)],
                        **prof, "oracle_ok": bool(ok)})
    eng.close()
    line = json.dumps({"workload": f"{n}-doc synthetic, {d}-d dense + Zipf BM25, hybrid rrf top_k={k}, {B}-query "
                                   "batches from host buffers",
                       "card": info, "steps": args.steps, "warmup": args.warmup, "results": results})
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")
    return 0 if all(r["oracle_ok"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
