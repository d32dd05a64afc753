"""K5 parity at weights whose attention is far from uniform (tests/ce_numerics.py): the reranker's logits and the
embedder's raw [CLS] states against the fp64 forward, within the tolerance the device-rounding emulation of the same case
predicts, over every attention kernel (S <= 128, 129..256, > 256), every hidden size, both residual streams and lengths
on both sides of every tile edge.  Then the batch structure of a forward pass (the prefix-sum carry past 1024 pairs, the
8-pair head groups, ``ce_stats``, slicing, workspace reuse) and ``rerank_dev`` across its 2048-pair chunk."""
import numpy as np
import pytest

import ce_numerics as cn
from oracle.cross_encoder import embed_from_cls

pytestmark = pytest.mark.gpu


def _load_reranker(engine, monkeypatch, w, stream):
    if stream == "fp32":
        monkeypatch.setenv("SB_CE_FP32_STREAM", "1")
    else:
        monkeypatch.delenv("SB_CE_FP32_STREAM", raising=False)
    engine.ce_load(w.blob(), w.config)


def _check(what, got, ref, emu, tol):
    got = np.asarray(got, np.float64)
    err, gap = np.abs(got - ref), np.abs(got - emu)
    line = f"{what}: max|gpu-fp64| {err.max():.3e}  max|gpu-emu| {gap.max():.3e}  tol {tol:.3e}"
    print(line)
    assert np.all(np.isfinite(got)) and err.max() <= tol, line


@pytest.mark.parametrize("stream", ["fp16", "fp32"])
@pytest.mark.parametrize("case", cn.RERANK_CASES, ids=lambda c: c.name)
def test_reranker_logits_match_fp64(engine, monkeypatch, case, stream):
    _load_reranker(engine, monkeypatch, case.weights(), stream)
    ids, tt, lens = cn.case_inputs(case)
    logits, sig = engine.ce_score(ids, tt, lens)
    _check(f"{case.name} {stream}", logits, cn.case_forward(case), cn.case_forward(case, stream),
           cn.case_tolerance(case, stream))
    assert np.allclose(sig, 1.0 / (1.0 + np.exp(-logits.astype(np.float64))), rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("case", cn.EMBED_CASES, ids=lambda c: c.name)
def test_embedder_cls_states_match_fp64(engine, case):
    w = case.weights()
    engine.enc_load(w.blob(), w.config)
    ids, tt, lens = cn.case_inputs(case)
    got = engine.enc_embed(ids, tt, lens, normalize=False)
    _check(case.name, got, cn.case_forward(case), cn.case_forward(case, "fp32"), cn.case_tolerance(case, "fp32"))


def test_embedder_projection_and_normalization_match_fp64(engine):
    case = cn.Case("embed", 384, 2, 300)
    w = case.weights()
    rng = np.random.default_rng(11)
    pw = (rng.standard_normal((256, 384)) / np.sqrt(384)).astype(np.float32)
    pb = (rng.standard_normal(256) * 0.1).astype(np.float32)
    engine.enc_load(w.blob(), w.config, pw, pb)
    ids, tt, lens = cn.case_inputs(case)
    got = engine.enc_embed(ids, tt, lens)
    ref = embed_from_cls(cn.case_forward(case), pw, pb)
    emu = embed_from_cls(cn.case_forward(case, "fp32"), pw, pb)
    _check(f"{case.name} projected", got, ref, emu, cn.tolerance(emu, ref))
    assert np.allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-5)


# ------------------------------------------------------------------------------------------------ batch structure
def _batch(P, S=64):
    """P pairs whose lengths cycle through the straddling lengths of S (0 and S + 9 included)."""
    lens = np.resize(np.asarray(cn.straddle_lengths(S), np.int32), P)
    return cn.token_inputs(S, lens, seed=P)


@pytest.mark.parametrize("P", [1, 7, 9, 1025, 2100])
def test_batch_sizes_match_fp64_and_count_stats(engine, monkeypatch, P):
    """P > 1024 carries ce_cu_kernel's prefix sum across blocks; P % 8 != 0 leaves a partial 8-pair head group."""
    w = cn.model_weights(128, 2)
    _load_reranker(engine, monkeypatch, w, "fp16")
    ids, tt, lens = _batch(P)
    engine.ce_stats(reset=True)
    logits, _ = engine.ce_score(ids, tt, lens)
    n = np.clip(lens, 1, ids.shape[1]).astype(np.int64)
    assert engine.ce_stats(reset=True) == (P, int(n.sum()), int((n * n).sum()))
    assert engine.ce_stats() == (0, 0, 0)
    ref = cn.forward(w, ids, tt, lens)[0]
    emu = cn.forward(w, ids, tt, lens, mode="fp16")[0]
    _check(f"batch P={P}", logits, ref, emu, cn.tolerance(emu, ref))


def test_slices_and_workspace_reuse_are_bit_identical(engine, monkeypatch):
    _load_reranker(engine, monkeypatch, cn.model_weights(128, 2), "fp16")
    ids, tt, lens = _batch(2100)
    full = engine.ce_score(ids, tt, lens)[0]
    cuts = [0, 1, 8, 17, 1042, 2100]
    parts = np.concatenate([engine.ce_score(ids[a:b], tt[a:b], lens[a:b])[0] for a, b in zip(cuts, cuts[1:])])
    assert np.array_equal(parts, full)
    small = engine.ce_score(ids[:7], tt[:7], lens[:7])[0]     # the large workspace, reused by a small pass
    again = engine.ce_score(ids, tt, lens)[0]
    assert np.array_equal(small, full[:7]) and np.array_equal(again, full)


# ------------------------------------------------------------------------------------------------ rerank_dev
def _frame_pairs(q_tok, q_len, cand, cnt, doc_tok, doc_len, id_base, S):
    """ce_build_pairs_kernel on the host: [CLS] query [SEP] doc [SEP] for every (query, candidate slot)."""
    B, k = cand.shape
    lq, ld = q_tok.shape[1], doc_tok.shape[1]
    ids = np.zeros((B * k, S), np.int32)
    tts = np.zeros((B * k, S), np.int32)
    lens = np.zeros(B * k, np.int32)
    for b in range(B):
        nq = min(max(int(q_len[b]), 0), min(lq, S // 2 - 2 if S // 2 - 2 > 0 else 1))
        for j in range(k):
            p = b * k + j
            ids[p, 0] = 101
            if j >= cnt[b]:
                ids[p, 1], lens[p] = 102, 2
                continue
            row = int(cand[b, j]) - id_base
            nd = min(int(doc_len[row]), ld) if 0 <= row < len(doc_len) else 0
            nd = max(min(nd, S - nq - 3), 0)
            ids[p, 1:nq + 1] = q_tok[b, :nq]
            ids[p, nq + 1] = 102
            if nd:
                ids[p, nq + 2:nq + 2 + nd] = doc_tok[row, :nd]
            ids[p, nq + 2 + nd] = 102
            tts[p, nq + 2:nq + 3 + nd] = 1
            lens[p] = nq + nd + 3
    return ids, tts, lens


def test_rerank_dev_across_the_2048_pair_chunk(engine, monkeypatch):
    import torch

    S, B, k, k_out, lq, ld, n_docs, id_base = 128, 24, 100, 40, 70, 150, 300, 1000
    rng = np.random.default_rng(21)
    _load_reranker(engine, monkeypatch, cn.model_weights(128, 2), "fp16")
    doc_tok = rng.integers(0, cn.VOCAB, (n_docs, ld)).astype(np.uint16)
    doc_len = rng.integers(0, 260, n_docs).astype(np.int32)        # beyond ld and beyond S - nq - 3
    doc_len[:3] = (0, ld, ld + 40)
    engine.ce_tokens_load(doc_tok, doc_len, id_base)
    q_tok = rng.integers(0, cn.VOCAB, (B, lq)).astype(np.int32)
    q_len = rng.integers(1, lq + 1, B).astype(np.int32)           # many longer than S / 2 - 2 = 62
    q_len[:4] = (lq + 5, 0, 62, 63)
    cand = rng.integers(id_base, id_base + n_docs, (B, k)).astype(np.int64)
    cand[3, 5:9] = (-1, id_base - 7, id_base + n_docs, id_base + n_docs + 1000)   # no such document: query only
    cand[4, [10, 50, 99]] = cand[4, 2]                              # duplicates: equal scores, stable order
    cand[5, :k:2] = cand[5, 1:k:2]
    cnt = np.full(B, k, np.int32)
    cnt[[0, 1, 2, 6]] = (0, 25, 77, 1)                               # none, fewer than k_out, fewer than k
    out_ids, out_sc, out_cnt = engine.rerank_dev(torch.from_numpy(q_tok).cuda(), torch.from_numpy(q_len).cuda(),
                                                 torch.from_numpy(cand).cuda(), torch.from_numpy(cnt).cuda(), S, k_out)
    torch.cuda.synchronize()
    out_ids, out_sc, out_cnt = out_ids.cpu().numpy(), out_sc.cpu().numpy(), out_cnt.cpu().numpy()
    ids, tts, lens = _frame_pairs(q_tok, q_len, cand, cnt, doc_tok, doc_len, id_base, S)
    assert lens.max() == S and np.all(lens[3 * k + 5:3 * k + 9] == 62 + 3)   # query 3: 62 tokens, no document
    sig = engine.ce_score(ids, tts, lens)[1].reshape(B, k)
    assert sig[4, 2] == sig[4, 10] == sig[4, 50] == sig[4, 99]
    for b in range(B):
        n = int(cnt[b])
        order = sorted(range(n), key=lambda j: (-sig[b, j], j))[:k_out]
        c = len(order)
        assert out_cnt[b] == c, b
        assert list(out_ids[b, :c]) == [int(cand[b, j]) for j in order], b
        assert np.allclose(out_sc[b, :c], sig[b, order], rtol=1e-5, atol=1e-6), b
        assert np.all(out_ids[b, c:] == -1) and np.all(out_sc[b, c:] == 0.0), b
