"""Recommendation by example (DESIGN.md K1j) on one GPU: 1 M x 1024 float16 Cosine, k = 100.  best_score and
sum_scores at 32 requests x 8 examples and 64 x 4, each alternated with a 256-query nearest batch of the same vectors
(the cost floor: one 256-column pass), plus average_vector.  Checks zero fallbacks and the fp64 oracle on a subset, and
writes records/bench_dense_reco_h100.json with the card's name and power limit read in the same run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=str(ROOT / "records" / "bench_dense_reco_h100.json"))
    a = ap.parse_args()
    from sentio_b200.engine import B200Engine
    from metric_oracle import stored_metric
    from reco_oracle import merged, similarities

    rng = np.random.default_rng(0)
    x = rng.standard_normal((a.n, a.d), dtype=np.float32)
    eng = B200Engine(0)
    eng.load_dense(x)
    ex = (x[rng.integers(0, a.n, 256)] + 0.3 * rng.standard_normal((256, a.d), dtype=np.float32)).astype(np.float32)
    k = 100
    res = {"card": card(), "n": a.n, "d": a.d, "k": k, "storage": "float16", "metric": "cosine", "workloads": {}}

    def timed(fn):
        fn()
        eng.sync()
        ts = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            fn()
            eng.sync()
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts))

    fb0 = eng.fallback_count()
    for R, m in ((32, 8), (64, 4)):
        r_off = np.arange(R + 1) * m
        n_pos = [m // 2 + 1] * R
        for strategy in ("best_score", "sum_scores"):
            t_reco, t_near = [], []
            for _ in range(3):   # alternated with the nearest batch of the same vectors
                t_reco.append(timed(lambda: eng.dense_recommend(ex, r_off, n_pos, [strategy] * R, k)))
                t_near.append(timed(lambda: eng.dense_topk(ex, k)))
            res["workloads"][f"{strategy}_{R}x{m}"] = {
                "ms_per_call": [round(t * 1e3, 3) for t in t_reco],
                "nearest_256_ms_per_call": [round(t * 1e3, 3) for t in t_near],
                "requests_per_s": round(R / float(np.median(t_reco)), 1)}
    qa = ex[:32]
    res["workloads"]["average_vector_32"] = {"ms_per_call": round(timed(lambda: eng.dense_topk(qa, k)) * 1e3, 3)}
    res["fallbacks"] = eng.fallback_count() - fb0
    # oracle on a subset: 2 requests of the 32 x 8 batch per strategy, similarities in fp64 on the stored fp16 rows,
    # computed in row chunks
    S = np.empty((a.n, 16))
    for c0 in range(0, a.n, 1 << 16):
        y = stored_metric(x[c0:c0 + (1 << 16)])[0].astype(np.float64)
        S[c0:c0 + len(y)] = np.stack([similarities(y, None, e, "cosine") for e in ex[:16]], 1)
    ok = True
    for strategy in ("best_score", "sum_scores"):
        ids, sc, cnt = eng.dense_recommend(ex[:16], [0, 8, 16], [5, 5], [strategy] * 2, k)
        for r in range(2):
            s_ = merged(S[:, 8 * r:8 * r + 8], 5, strategy)
            wi = np.lexsort((np.arange(a.n), -s_))[:k]
            ok &= bool(np.array_equal(ids[r, :cnt[r]], wi)) and bool(np.allclose(sc[r, :cnt[r]], s_[wi], rtol=1e-9))
    res["oracle_subset_ok"] = ok
    eng.close()
    Path(a.out).write_text(json.dumps(res) + "\n")
    print(json.dumps(res))
    return 0 if ok and res["fallbacks"] == 0 else 1


if __name__ == "__main__":
    sys.exit(main())
