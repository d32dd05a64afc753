#!/usr/bin/env python
"""Small filtered dense workload for `compute-sanitizer` (memcheck / racecheck): the match-mask kernel, the
low-cardinality gather path, the masked CUDA-core and wgmma scans, and the brute-force fallback (exact duplicates
inside the matching set, the zero query), checked against the oracle."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from oracle import dense as dense_oracle
    from sentio_b200.engine import B200Engine

    eng = B200Engine(0)
    rng = np.random.default_rng(2)
    n, d, k = 12_000, 128, 20
    x = rng.standard_normal((n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x16 = x.astype(np.float16)
    x16[3000:5600] = x16[11]                          # 2600 duplicates inside field 0 == 1: brute-force fallback
    tag0 = np.where(rng.random(n) < 0.4, 0, 1).astype(np.int32)
    tag0[3000:5600] = 1
    tag0[11] = 1
    tag1 = (np.arange(n) % 50).astype(np.int32)       # 240 rows per value: the gather path
    eng.load_dense(x16)
    eng.load_dense_tags(0, tag0)
    eng.load_dense_tags(1, tag1)
    tags = [tag0, tag1]
    cases = [[(0, 0)], [(0, 1)], [(1, 7)], [(0, 0), (1, 3)], [], [(1, 99)]]
    for mode, B in ((1, 3), (0, 40), (0, 130), (0, 256), (0, 300)):
        eng.dense_set_mode(mode)
        q = rng.standard_normal((B, d)).astype(np.float32)
        q[1] = x16[11].astype(np.float32)
        q[2] = 0.0
        conds = [cases[b % len(cases)] for b in range(B)]
        conds[1] = [(0, 1)]
        off = np.zeros(B + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in conds])
        fld = np.asarray([f for c in conds for f, _ in c], np.int32)
        code = np.asarray([v for c in conds for _, v in c], np.int32)
        ids, sc, cnt = eng.dense_topk(q, k, filters=(off, fld, code))
        for b in range(B):
            m = np.ones(n, bool)
            for f, v in conds[b]:
                m &= tags[f] == v
            idx = np.flatnonzero(m)
            wi, ws = dense_oracle.dense_topk(x16[idx], q[b], k)
            assert list(ids[b, :cnt[b]]) == list(idx[wi]) and np.allclose(sc[b, :cnt[b]], ws, rtol=1e-9, atol=1e-12), \
                (B, b)
        print("mode", mode, "B =", B, "ok", flush=True)
    eng.dense_set_mode(0)
    print("fallbacks:", eng.fallback_count(), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
