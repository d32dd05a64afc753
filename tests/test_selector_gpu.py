"""K7 parity: sb_select_dev (batched device selector) == sentio_b200.selector.select_documents, the host mirror that is
itself pinned to the reference's select_documents_node by tests/golden/selector.json."""
import numpy as np
import pytest

from sentio_b200.document import Document
from sentio_b200.selector import select_documents, selector_chars

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_select_dev_matches_host_selector(engine, dtype):
    import torch

    rng = np.random.default_rng(5)
    n_docs, B, k = 500, 64, 40
    docs = []
    for i in range(n_docs):
        r = rng.random()
        text = "x" * int(rng.integers(1, 600)) if r < 0.8 else ("" if r < 0.9 else "  ")
        meta = {"content": "c" * int(rng.integers(0, 300))} if rng.random() < 0.5 else {}
        docs.append(Document(id=str(i), text=text, metadata=meta))
    engine.load_doc_chars(np.array([selector_chars(d) for d in docs], np.int32), id_base=1000)
    cand = rng.integers(0, n_docs, size=(B, k))           # repeated ids inside a query
    scores = np.round(rng.random((B, k)), 1).astype(dtype)  # ties -> the stable order matters
    cnt = rng.integers(0, k + 1, size=B).astype(np.int32)
    for top_k, max_tokens in [(3, 2000), (10, 300), (40, 100000), (5, 0)]:
        out = engine.select_dev(torch.from_numpy(cand + 1000).cuda(), torch.from_numpy(scores).cuda(),
                                torch.from_numpy(cnt).cuda(), top_k, max_tokens)
        torch.cuda.synchronize()
        ids, sc, n_sel, toks = [t.cpu().numpy() for t in out]
        for b in range(B):
            cands = []
            for j in range(int(cnt[b])):
                d = docs[int(cand[b, j])]
                cands.append(Document(id=d.id, text=d.text, metadata={**d.metadata, "score": float(scores[b, j])}))
            want, want_tokens = select_documents(cands, top_k, max_tokens)
            assert int(n_sel[b]) == len(want) and int(toks[b]) == want_tokens, (b, top_k, max_tokens)
            assert [str(int(i) - 1000) for i in ids[b, :n_sel[b]]] == [d.id for d in want]
            assert [float(x) for x in sc[b, :n_sel[b]]] == [d.metadata["score"] for d in want]
            assert np.all(ids[b, n_sel[b]:] == -1)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_select_dev_at_the_shared_memory_limit(engine, dtype):
    """k = 4094 candidates (the 48 KB limit of the per-query sort), top_k >= k, and candidate ids outside the loaded
    doc_chars range, which the selector treats as blank documents."""
    import torch

    rng = np.random.default_rng(6)
    n_docs, base, B, k = 500, 1000, 5, 4094
    chars = rng.integers(0, 600, n_docs).astype(np.int32)
    chars[rng.random(n_docs) < 0.1] = 0
    engine.load_doc_chars(chars, id_base=base)
    cand = rng.integers(base - 20, base + n_docs + 20, size=(B, k)).astype(np.int64)   # some outside the range
    cand[:, :4] = [0, -1, base - 1, base + n_docs]
    scores = np.round(rng.random((B, k)), 2).astype(dtype)
    scores[:, :4] = 2.0                                    # the out-of-range ids are walked first
    cnt = np.asarray([k, k - 1, 4000, 17, 0], np.int32)
    inside = (cand >= base) & (cand < base + n_docs)
    assert (~inside[:, :4]).all() and (~inside[:, 4:]).any()

    def text_of(i):
        return "x" * int(chars[i - base]) if base <= i < base + n_docs else ""

    for top_k, max_tokens in [(k, 10 ** 8), (5000, 10 ** 8), (4100, 3000)]:
        out = engine.select_dev(torch.from_numpy(cand).cuda(), torch.from_numpy(scores).cuda(),
                                torch.from_numpy(cnt).cuda(), top_k, max_tokens)
        torch.cuda.synchronize()
        ids, sc, n_sel, toks = [t.cpu().numpy() for t in out]
        for b in range(B):
            cands = [Document(id=str(int(cand[b, j])), text=text_of(int(cand[b, j])),
                              metadata={"score": float(scores[b, j])}) for j in range(int(cnt[b]))]
            want, want_tokens = select_documents(cands, top_k, max_tokens)
            assert int(n_sel[b]) == len(want) and int(toks[b]) == want_tokens, (b, top_k, max_tokens)
            assert [str(int(i)) for i in ids[b, :n_sel[b]]] == [d.id for d in want]
            assert [float(x) for x in sc[b, :n_sel[b]]] == [d.metadata["score"] for d in want]
            assert np.all(ids[b, n_sel[b]:] == -1)
            assert not set(ids[b, :n_sel[b]].tolist()) & {0, -1, base - 1, base + n_docs}


def test_select_dev_beyond_the_shared_memory_limit_is_unsupported(engine):
    import torch

    from sentio_b200._lib import SentioB200Error

    engine.load_doc_chars(np.ones(10, np.int32))
    k = 4095
    with pytest.raises(SentioB200Error, match=r"rc=-4\).*too large"):
        engine.select_dev(torch.zeros((1, k), dtype=torch.int64, device="cuda"),
                          torch.zeros((1, k), dtype=torch.float32, device="cuda"),
                          torch.zeros(1, dtype=torch.int32, device="cuda"), 3, 100)
