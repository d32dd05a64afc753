#!/usr/bin/env python
"""Small dense workload for `compute-sanitizer` (memcheck / racecheck): the wgmma scan (one group, a 256-query group plus
a small one, two 256-query groups), the CUDA-core scan, the window select + exact re-score and the brute-force fallback,
checked against the oracle."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from oracle import dense as dense_oracle
    from sentio_b200.engine import B200Engine

    eng = B200Engine(0)
    rng = np.random.default_rng(1)
    n, d, k = 12_000, 128, 20
    x = rng.standard_normal((n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x16 = x.astype(np.float16)
    x16[3000:5600] = x16[11]                     # 2600 exact duplicates: window > winner buffer -> brute-force fallback
    eng.load_dense(x16)
    for B in (3, 40, 130, 256, 300, 512):             # CUDA-core scan / one wgmma group / a full group (+ a small one) / two
        q = rng.standard_normal((B, d)).astype(np.float32)
        q[1] = x16[11].astype(np.float32)
        q[2] = 0.0
        ids, sc, cnt = eng.dense_topk(q, k)
        for b in range(B):
            wi, ws = dense_oracle.dense_topk(x16, q[b], k)
            assert list(ids[b]) == list(wi) and np.allclose(sc[b], ws, rtol=1e-9, atol=1e-12), (B, b)
        print("B =", B, "ok", flush=True)
    eng.close()


if __name__ == "__main__":
    main()
