"""K5 parity: wgmma GEMM unit test, cross-encoder forward vs the NumPy / HuggingFace oracles (sigmoid: rel 1e-3, abs
floor 1e-4; logits: the device-emulation tolerance of tests/ce_numerics.py), and the reranker's control flow vs the reference JinaReranker (golden rerank_flow.json)."""
import math

import numpy as np
import pytest

import ce_numerics as cn
from conftest import load_golden
from oracle import cross_encoder as ce_oracle
from sentio_b200 import synth
from sentio_b200.cross_encoder import MINILM_L6, CrossEncoderWeights
from sentio_b200.document import Document
from sentio_b200.index import hash_tokenize_pairs

pytestmark = pytest.mark.gpu

_erf = np.vectorize(math.erf)


@pytest.mark.parametrize("M,N,K,epi", [(128, 128, 64, 0), (200, 256, 384, 0), (1000, 1152, 384, 0), (333, 1536, 384, 1),
                                       (512, 384, 1536, 2), (77, 128, 128, 2),
                                       # >= 4 row tiles and K <= 384 -> weight-stationary persistent kernel
                                       (2048, 384, 384, 2), (5000, 1536, 384, 1), (700, 128, 64, 0), (25600, 1152, 384, 0),
                                       (513, 256, 192, 2),
                                       (2304, 640, 192, 0), (4100, 512, 384, 1), (9000, 1152, 384, 0), (2048, 1536, 128, 1),
                                       # epi 3: the fp16 residual stream (residual operand and output in fp16)
                                       (96, 384, 384, 3), (700, 384, 1536, 3), (3000, 384, 384, 3), (2600, 384, 1536, 3),
                                       # hidden 768 (QKV, FFN up, FFN down on both streams) and hidden 256 (QKV)
                                       *[(M, N, K, epi) for (N, K, epi) in ((2304, 768, 0), (3072, 768, 1), (768, 3072, 2),
                                                                            (768, 3072, 3), (768, 256, 0))
                                         for M in (1, 127, 129)]])
def test_tcgen05_gemm_matches_numpy(engine, M, N, K, epi):
    rng = np.random.default_rng(M + N + K + epi)
    a = rng.standard_normal((M, K)).astype(np.float32)
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32) * 0.1
    res = rng.standard_normal((M, N)).astype(np.float32) if epi in (2, 3) else None
    got = engine.ce_gemm_test(a, w, bias, epi, res)
    a16 = a.astype(np.float16).astype(np.float64)
    w16 = w.astype(np.float16).astype(np.float64)
    want = a16 @ w16.T + bias
    if epi == 1:
        want = 0.5 * want * (1.0 + _erf(want / math.sqrt(2.0)))
    if epi == 3:
        want = want + res.astype(np.float16).astype(np.float64)
    if epi == 2:
        want = want + res
        assert np.allclose(got, want, rtol=1e-4, atol=1e-4)
    else:
        assert np.allclose(got, want.astype(np.float16).astype(np.float64), rtol=2e-3, atol=2e-3)


def _pairs(n_docs, seq_len=128):
    flat, off = synth.text_corpus_tokens(n_docs, vocab=4000)
    docs = synth.texts_from_tokens(flat, off)
    docs[1] = ""           # empty document
    docs[2] = "w1 " * 400   # longer than the window -> truncated
    return hash_tokenize_pairs("w1 w5 w9 w100 w3 w7", docs, seq_len)


def _assert_logits_within_emulated_tolerance(w, ids, tt, lens, logits):
    """|logit - fp64| within 3 x the distance of the device-rounding emulation (fp16 residual stream, the reranker's
    default) from fp64, plus 1e-5 (tests/ce_numerics.py)."""
    ref = cn.forward(w, ids, tt, lens)[0]
    tol = cn.tolerance(cn.forward(w, ids, tt, lens, mode="fp16")[0], ref)
    err = np.abs(logits.astype(np.float64) - ref).max()
    assert err <= tol, f"max|gpu-fp64| {err:.3e} > tol {tol:.3e}"


def test_small_model_vs_numpy_oracle(engine):
    cfg = dict(vocab_size=30522, hidden=128, layers=2, heads=4, intermediate=256, max_pos=128, type_vocab=2, ln_eps=1e-12)
    w = CrossEncoderWeights.random(cfg, seed=3, std=0.05)
    engine.ce_load(w.blob(), cfg)
    ids, tt, lens = _pairs(9, 64)
    logits, sig = engine.ce_score(ids, tt, lens)
    want_l, want_s = ce_oracle.numpy_forward(w, ids, tt, lens)
    assert np.allclose(sig, want_s, rtol=1e-3, atol=1e-4)
    assert np.allclose(logits, want_l, rtol=1e-2, atol=2e-3)
    _assert_logits_within_emulated_tolerance(w, ids, tt, lens, logits)


@pytest.mark.parametrize("seq_len", [200, 256, 320])
def test_windows_longer_than_128_tokens(engine, seq_len):
    """128 < S <= 256 runs the 256-key tensor-core attention (8 query tiles per warp pair), S > 256 the generic kernel;
    every query row of a long pair must be attended (round 1 only covered the first 128 rows of the 256-key variant)."""
    cfg = dict(vocab_size=30522, hidden=128, layers=2, heads=4, intermediate=256, max_pos=512, type_vocab=2, ln_eps=1e-12)
    w = CrossEncoderWeights.random(cfg, seed=5, std=0.1)   # scores spread over 0.45 .. 0.73 (std 0.05: all ~0.547)
    engine.ce_load(w.blob(), cfg)
    flat, off = synth.text_corpus_tokens(40, vocab=4000)
    docs = synth.texts_from_tokens(flat, off)
    long_docs = [" ".join(docs[i:i + 1 + i % 5]) for i in range(0, 30, 2)] + ["", "w1 " * 600]
    ids, tt, lens = hash_tokenize_pairs("w1 w5 w9 w100 w3 w7", long_docs, seq_len)
    assert int(lens.max()) == seq_len and int((lens > 128).sum()) >= 4 and int((lens < 128).sum()) >= 2
    logits, sig = engine.ce_score(ids, tt, lens)
    want_l, want_s = ce_oracle.numpy_forward(w, ids, tt, lens)
    assert want_s.max() - want_s.min() > 0.2
    assert np.allclose(sig, want_s, rtol=2e-3, atol=2e-4), np.abs(sig - want_s).max()   # 5 x the init scale of the path's test
    _assert_logits_within_emulated_tolerance(w, ids, tt, lens, logits)


def test_minilm_l6_vs_huggingface_oracle(engine):
    model = ce_oracle.hf_model(MINILM_L6, seed=0)
    w = CrossEncoderWeights.from_hf_state_dict(model.state_dict(), MINILM_L6)
    engine.ce_load(w.blob(), MINILM_L6)
    ids, tt, lens = _pairs(24, 128)
    logits, sig = engine.ce_score(ids, tt, lens)
    want_l, want_s = ce_oracle.hf_scores(model, ids, tt, lens)
    assert np.all((sig >= 0) & (sig <= 1))  # Source.score in [0, 1] (reference api/app.py:157)
    assert np.allclose(sig, want_s, rtol=1e-3, atol=1e-4), np.abs(sig - want_s).max()
    # the fp64 forward of the same weights (pinned to HuggingFace on the CPU) at the device-emulation tolerance
    _assert_logits_within_emulated_tolerance(w, ids, tt, lens, logits)
    # batch-size independence: 100 pairs in one call == the same pairs in slices
    ids2, tt2, lens2 = _pairs(100, 128)
    a = engine.ce_score(ids2, tt2, lens2)[1]
    b = np.concatenate([engine.ce_score(ids2[i:i + 33], tt2[i:i + 33], lens2[i:i + 33])[1] for i in range(0, 100, 33)])
    assert np.array_equal(a, b)


def test_reranker_control_flow_matches_reference(engine):
    from sentio_b200.rerankers.b200_reranker import B200Reranker

    cfg = dict(vocab_size=30522, hidden=128, layers=1, heads=4, intermediate=128, max_pos=128, type_vocab=2, ln_eps=1e-12)
    rr = B200Reranker(weights=CrossEncoderWeights.random(cfg, seed=1), engine=engine, seq_len=64)
    assert rr.rerank("q", [], top_k=3) == []
    for c in load_golden("rerank_flow"):
        docs = [Document(id=f"r{i}", text=(f"text {i}" if i % 4 else ""), metadata={"content": f"fallback {i}"})
                for i in range(c["n"])]
        if c["kind"] == "scores":
            rr.score_pairs = lambda q, texts, rel=c["rel"]: np.asarray(rel)  # canned relevance, like the golden run
            out = rr.rerank("some query", docs, top_k=c["top_k"])
        else:
            docs = [Document(id=f"r{i}", text=f"text {i}", metadata={"score": 0.5}) for i in range(c["n"])]
            out = rr.rerank("   ", docs, top_k=c["top_k"])
        got = [[d.id, d.metadata["rerank_score"], d.metadata["score"], d.text] for d in out]
        assert got == c["expected"], c
    # real scoring path: sorted descending, scores in [0,1], never raises
    del rr.score_pairs
    docs = [Document(id=str(i), text=f"w{i} w{i+1} w{i+2}") for i in range(20)]
    out = rr.rerank("w3 w4", docs, top_k=5)
    s = [d.metadata["rerank_score"] for d in out]
    assert len(out) == 5 and s == sorted(s, reverse=True) and all(0 <= x <= 1 for x in s)
    rr._engine = None  # force a failure inside rerank -> default ranking, no exception
    out = rr.rerank("w3 w4", docs, top_k=3)
    assert [d.id for d in out] == ["0", "1", "2"] and [d.metadata["rerank_score"] for d in out] == [1.0, 0.9, 0.8]


def test_batched_rerank_pipeline_equals_per_query_reranker(engine):
    """sb_rerank_dev (device-side pair framing + cross-encoder + ranking) == hash_tokenize_pairs + sb_ce_score per query."""
    from sentio_b200.index import build_bm25_from_token_ids, doc_token_matrix, hash_vocab_ids
    from sentio_b200.pipeline import HybridPipeline

    n, d, k, k_out, B, V = 9000, 128, 40, 10, 5, 3000
    x = synth.dense_corpus(n, d)
    flat, off = synth.text_corpus_tokens(n, vocab=V)
    idx = build_bm25_from_token_ids(flat, off)
    vocab_ids = hash_vocab_ids(V)
    doc_tok, doc_len = doc_token_matrix(flat, off, vocab_ids, ld=120)
    cfg = dict(vocab_size=30522, hidden=128, layers=2, heads=4, intermediate=256, max_pos=128, type_vocab=2, ln_eps=1e-12)
    w = CrossEncoderWeights.random(cfg, seed=5, std=0.05)
    pipe = HybridPipeline(0)
    pipe.load_dense(x)
    pipe.load_bm25(idx)
    pipe.load_cross_encoder(w)
    pipe.load_doc_tokens(doc_tok, doc_len)
    q = synth.query_vectors(B, d)
    q_raw = synth.query_tokens(B, vocab=V)
    terms = [idx.term_ids(t) for t in q_raw]
    q_tok = vocab_ids[q_raw].astype(np.int32)
    q_len = np.full(B, q_raw.shape[1], np.int32)
    ids, sc, cnt = pipe.search_hybrid_rerank(q, terms, q_tok, q_len, k, k_out, seq_len=128)
    f_ids, f_sc, f_src, f_cnt = pipe.search_hybrid(q, terms, k)
    engine.ce_load(w.blob(), cfg)
    texts = synth.texts_from_tokens(flat, off)
    for b in range(B):
        cand = [int(i) for i in f_ids[b, :f_cnt[b]]]
        pi, pt, pl = hash_tokenize_pairs(synth.token_text(q_raw[b]), [texts[i] for i in cand], 128)
        _, sig = engine.ce_score(pi, pt, pl)
        order = sorted(range(len(cand)), key=lambda j: -sig[j])[:k_out]  # stable, like the reference's sorted()
        assert [int(i) for i in ids[b, :cnt[b]]] == [cand[j] for j in order]
        assert np.allclose(sc[b, :cnt[b]], sig[order], rtol=1e-5, atol=1e-6)
