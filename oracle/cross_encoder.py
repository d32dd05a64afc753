"""Cross-encoder oracle (TEST INFRASTRUCTURE).

The reference has no local cross-encoder (README.md:63; src/core/rerankers/jina_reranker.py:139 posts to a hosted model),
so BASELINE.json config 4 defines the scorer: a random-init MiniLM-L6-shaped ``BertForSequenceClassification``
(num_labels=1), relevance = sigmoid(logit).  Two oracles:

* ``hf_model`` / ``hf_scores``  -- HuggingFace transformers (library code shipped in the image), fp32 on CPU.
* ``numpy_forward``             -- our own fp32/fp64 NumPy restatement of the same forward pass (post-LN BERT, erf-GELU,
  additive -inf style attention mask, pooler tanh on [CLS], linear classifier); tests pin it against ``hf_scores``.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.special import erf as _erf


def hf_model(cfg: dict, seed: int = 0):
    import torch
    from transformers import BertConfig, BertForSequenceClassification

    torch.manual_seed(seed)
    bc = BertConfig(vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden"], num_hidden_layers=cfg["layers"],
                    num_attention_heads=cfg["heads"], intermediate_size=cfg["intermediate"],
                    max_position_embeddings=cfg["max_pos"], type_vocab_size=cfg.get("type_vocab", 2), num_labels=1,
                    hidden_act="gelu", layer_norm_eps=cfg.get("ln_eps", 1e-12), hidden_dropout_prob=0.0,
                    attention_probs_dropout_prob=0.0)
    model = BertForSequenceClassification(bc)
    model.eval()
    return model


def hf_scores(model, input_ids, token_type, lengths, batch: int = 32):
    import torch

    ids = torch.as_tensor(np.asarray(input_ids), dtype=torch.long)
    tt = torch.as_tensor(np.asarray(token_type), dtype=torch.long)
    S = ids.shape[1]
    mask = (torch.arange(S)[None, :] < torch.as_tensor(np.asarray(lengths), dtype=torch.long)[:, None]).long()
    out = []
    with torch.no_grad():
        for i in range(0, ids.shape[0], batch):
            o = model(input_ids=ids[i:i + batch], token_type_ids=tt[i:i + batch], attention_mask=mask[i:i + batch])
            out.append(o.logits.reshape(-1).double())
    logits = torch.cat(out).numpy() if out else np.zeros(0)
    return logits, 1.0 / (1.0 + np.exp(-logits))


def _ln(x, g, b, eps):
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * g + b


def _gelu(x):
    return 0.5 * x * (1.0 + _erf(x / math.sqrt(2.0)))


def numpy_forward(weights, input_ids, token_type, lengths, dtype=np.float64):
    """weights: sentio_b200.cross_encoder.CrossEncoderWeights (plain name->array container)."""
    cfg, t = weights.config, {k: v.astype(dtype) for k, v in weights.tensors.items()}
    H, L, NH, eps = cfg["hidden"], cfg["layers"], cfg["heads"], cfg.get("ln_eps", 1e-12)
    dh = H // NH
    ids, tt = np.asarray(input_ids), np.asarray(token_type)
    P, S = ids.shape
    x = t["word_emb"][ids] + t["pos_emb"][np.arange(S)][None] + t["type_emb"][tt]
    x = _ln(x, t["emb_ln_g"], t["emb_ln_b"], eps)
    mask = np.arange(S)[None, :] < np.asarray(lengths)[:, None]
    bias = np.where(mask, 0.0, np.finfo(np.float32).min)[:, None, None, :]
    for l in range(L):
        p = f"l{l}."
        q = (x @ t[p + "wq"].T + t[p + "bq"]).reshape(P, S, NH, dh).transpose(0, 2, 1, 3)
        k = (x @ t[p + "wk"].T + t[p + "bk"]).reshape(P, S, NH, dh).transpose(0, 2, 1, 3)
        v = (x @ t[p + "wv"].T + t[p + "bv"]).reshape(P, S, NH, dh).transpose(0, 2, 1, 3)
        s = q @ k.transpose(0, 1, 3, 2) / math.sqrt(dh) + bias
        s = s - s.max(-1, keepdims=True)
        e = np.exp(s)
        a = e / e.sum(-1, keepdims=True)
        ctx = (a @ v).transpose(0, 2, 1, 3).reshape(P, S, H)
        x = _ln(ctx @ t[p + "wo"].T + t[p + "bo"] + x, t[p + "ln1_g"], t[p + "ln1_b"], eps)
        h = _gelu(x @ t[p + "w1"].T + t[p + "b1"])
        x = _ln(h @ t[p + "w2"].T + t[p + "b2"] + x, t[p + "ln2_g"], t[p + "ln2_b"], eps)
    pooled = np.tanh(x[:, 0] @ t["pool_w"].T + t["pool_b"])
    logits = pooled @ t["cls_w"] + t["cls_b"][0]
    return logits, 1.0 / (1.0 + np.exp(-logits))


# ------------------------------------------------------------------------------------------------ embedder oracle
def hf_cls_states(model, input_ids, token_type, lengths, batch: int = 32):
    """Final-layer [CLS] hidden states of the BERT encoder inside ``model`` (fp32 CPU), shape [P, H] -- the oracle of the
    on-device query embedder (SURVEY.md 8f row 1): the encoder stack is the cross-encoder's, pinned above."""
    import torch

    ids = torch.as_tensor(np.asarray(input_ids), dtype=torch.long)
    tt = torch.as_tensor(np.asarray(token_type), dtype=torch.long)
    S = ids.shape[1]
    mask = (torch.arange(S)[None, :] < torch.as_tensor(np.asarray(lengths), dtype=torch.long)[:, None]).long()
    out = []
    with torch.no_grad():
        for i in range(0, ids.shape[0], batch):
            o = model.bert(input_ids=ids[i:i + batch], token_type_ids=tt[i:i + batch], attention_mask=mask[i:i + batch])
            out.append(o.last_hidden_state[:, 0].double())
    return torch.cat(out).numpy() if out else np.zeros((0, 0))


def embed_from_cls(cls_states, proj_w=None, proj_b=None, normalize=True):
    """embedding = normalize(W_proj cls + b_proj)  (fp64)."""
    y = np.asarray(cls_states, dtype=np.float64)
    if proj_w is not None:
        y = y @ np.asarray(proj_w, dtype=np.float64).T + np.asarray(proj_b, dtype=np.float64)
    if normalize:
        n = np.linalg.norm(y, axis=1, keepdims=True)
        y = y / np.where(n > 0, n, 1.0)
    return y
