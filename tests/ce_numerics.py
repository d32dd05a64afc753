"""Cross-encoder numerics for the K5 parity tests (TEST INFRASTRUCTURE, DESIGN.md K5).

Three things, shared by tests/test_ce_numerics_cpu.py and tests/test_ce_numerics_gpu.py:

* ``forward(..., mode="fp64")`` -- the fp64 forward of ``oracle.cross_encoder.numpy_forward`` on the device's packed
  layout: pair p holds ``clamp(len[p], 1, S)`` tokens (``ce_cu_kernel``), and the last layer runs for the [CLS] row only.
  ``defect=`` seeds one attention / [CLS]-tail fault into this CPU forward (nothing is injected into the library), so
  the tests can show that their tolerance would see it (``DEFECTS``).
* ``forward(..., mode="fp16" | "fp32")`` -- the same forward with the device's rounding points (``ce_forward``): fp16
  GEMM weights and outputs, fp16 probabilities as the A operand of P V in the tensor-core attention (S <= 256; the row
  sum stays unrounded, the generic S > 256 kernel and the [CLS] kernel keep them fp32), the packed-half GELU of
  ``ce_gemm.cu`` (``gelu_erf_h2``), and either residual stream: "fp16" rounds the pre-LayerNorm sums and the LayerNorm
  outputs (the reranker's default), "fp32" keeps them (``SB_CE_FP32_STREAM=1``, the embedder).  The last layer's [CLS]
  tail is fp32 in both.  Left out: fp32 accumulation order, ex2.approx / __expf, tanh.approx's own error.
* ``tolerance(emu, ref)`` -- the one tolerance rule: 3 x the emulation's largest distance from fp64, plus 1e-5.  It
  applies to the logit of every pair (reranker) or to every element of the raw [CLS] state (embedder).

The case table (``RERANK_CASES``, ``EMBED_CASES``) lives here so that the CPU power check and the GPU comparison run on
the same weights: ``std = sqrt(1.4 / H)`` puts the attention scores of every head at a standard deviation near 1.4, so a
wrong softmax moves the output far beyond the tolerance (weights near HuggingFace's N(0, 0.02) init leave attention
almost uniform, and a uniform average would pass a fixed 1e-3 tolerance).
"""
from __future__ import annotations

import functools
import math
import zlib
from dataclasses import dataclass

import numpy as np

from oracle.cross_encoder import _gelu, _ln
from sentio_b200.cross_encoder import CrossEncoderWeights

DH = 32            # head dimension: sb_ce_load requires it
VOCAB = 2048
TOL_FACTOR = 3.0
TOL_FLOOR = 1e-5
DEFECTS = ("uniform_attention", "drop_last_key", "admit_masked_key", "no_scale", "next_head_v", "next_pair_residual")

# packed-half GELU of ce_gemm.cu: gelu(x) ~ 0.5 x (1 + tanh(x (c0 + c1 x^2 + c2 x^4))), scripts/fit_gelu.py
_GELU_C0, _GELU_C1, _GELU_C2 = (np.float16(c) for c in (0.79745847075, 0.0370503451315, -0.00035873236644))


def r16(a):
    """Round to fp16 and back, through fp32 as the device does (fp64 in, fp64 out)."""
    with np.errstate(over="ignore"):
        return np.asarray(a, np.float64).astype(np.float32).astype(np.float16).astype(np.float64)


def gelu_fp16(x16):
    """``gelu_erf_h2`` on fp16 inputs: every packed-half operation rounds to fp16 once (an FMA once, not twice)."""
    x = np.asarray(x16, np.float64)
    x2 = np.minimum(r16(x * x), 36.0)
    q = r16(float(_GELU_C2) * x2 + float(_GELU_C1))
    q = r16(q * x2 + float(_GELU_C0))
    t = r16(np.tanh(r16(x * q)))
    hx = r16(0.5 * x)
    return r16(hx * t + hx)


def tolerance(emu, ref) -> float:
    """The tolerance of a case: 3 x max |emulation - fp64| over its pairs (or [CLS] elements), plus 1e-5."""
    return TOL_FACTOR * float(np.max(np.abs(np.asarray(emu, np.float64) - np.asarray(ref, np.float64)))) + TOL_FLOOR


# ------------------------------------------------------------------------------------------------ forward
_prepared: dict = {}


def _prepare(weights):
    """(fp64 tensors, fp16-rounded GEMM weights) of a weights object, kept for the last few objects used."""
    hit = _prepared.get(id(weights))
    if hit is not None and hit[0] is weights:
        return hit[1], hit[2]
    t = {k: np.asarray(v, np.float64) for k, v in weights.tensors.items()}
    w16 = {k: r16(v) for k, v in t.items() if k.split(".")[-1] in ("wq", "wk", "wv", "wo", "w1", "w2")}
    if len(_prepared) >= 3:
        _prepared.pop(next(iter(_prepared)))
    _prepared[id(weights)] = (weights, t, w16)
    return t, w16


def _attend(q, k, v, S, defect, round_p):
    """Masked softmax attention of one pair: q [nq, H] against the pair's n valid keys k, v [n, H]."""
    nq, H = q.shape
    n, nh = k.shape[0], H // DH
    qh = q.reshape(nq, nh, DH).transpose(1, 0, 2)
    kh = k.reshape(n, nh, DH).transpose(1, 0, 2)
    vh = v.reshape(n, nh, DH).transpose(1, 0, 2)
    if defect == "next_head_v":
        vh = np.roll(vh, -1, axis=0)                      # head h reads head h + 1's values
    elif defect == "drop_last_key" and n > 1:
        kh, vh = kh[:, :-1], vh[:, :-1]
    elif defect == "admit_masked_key" and n < S:          # the padding key: zero-filled K and V rows
        z = np.zeros((nh, 1, DH))
        kh, vh = np.concatenate([kh, z], axis=1), np.concatenate([vh, z], axis=1)
    s = qh @ kh.transpose(0, 2, 1)
    if defect == "uniform_attention":
        s = np.zeros_like(s)
    elif defect != "no_scale":
        s = s / math.sqrt(DH)
    e = np.exp(s - s.max(-1, keepdims=True))
    ctx = ((r16(e) if round_p else e) @ vh) / e.sum(-1, keepdims=True)
    return ctx.transpose(1, 0, 2).reshape(nq, H)


def forward(weights, input_ids, token_type, lengths, mode="fp64", defect=None):
    """(logits [P], final [CLS] states [P, H]) of the cross-encoder in fp64 (``mode="fp64"``) or under the device's
    rounding with the fp16 / fp32 residual stream (``mode="fp16"`` / ``"fp32"``); see the module docstring."""
    assert mode in ("fp64", "fp16", "fp32") and (defect is None or defect in DEFECTS)
    cfg = weights.config
    H, NL, eps = cfg["hidden"], cfg["layers"], cfg.get("ln_eps", 1e-12)
    assert cfg["heads"] * DH == H
    t, w16 = _prepare(weights)
    emu = mode != "fp64"
    rd = r16 if emu else (lambda a: a)
    act = (lambda a: gelu_fp16(r16(a))) if emu else _gelu

    def W(name):  # GEMM weights are stored in fp16 on the device
        return w16[name] if emu else t[name]

    ids, tts = np.asarray(input_ids), np.asarray(token_type)
    P, S = ids.shape
    n = np.clip(np.asarray(lengths, np.int64), 1, S)
    cu = np.concatenate([[0], np.cumsum(n)])
    pair = np.repeat(np.arange(P), n)
    pos = np.arange(cu[-1]) - cu[pair]
    x = t["word_emb"][ids[pair, pos]] + t["pos_emb"][pos] + t["type_emb"][tts[pair, pos]]
    res = _ln(x, t["emb_ln_g"], t["emb_ln_b"], eps)       # residual stream
    if mode == "fp16":
        res = r16(res)
    x16 = rd(res)                                          # GEMM operand
    for layer in range(NL):
        p = f"l{layer}."
        last = layer == NL - 1
        k = rd(x16 @ W(p + "wk").T + t[p + "bk"])
        v = rd(x16 @ W(p + "wv").T + t[p + "bv"])
        q = rd((x16[cu[:-1]] if last else x16) @ W(p + "wq").T + t[p + "bq"])
        # the tensor-core kernels (S <= 256) pack the probabilities to fp16 for P V; the others keep them fp32
        round_p = emu and not last and S <= 256
        ctx = np.concatenate([_attend(q[i:i + 1] if last else q[cu[i]:cu[i + 1]], k[cu[i]:cu[i + 1]],
                                      v[cu[i]:cu[i + 1]], S, defect, round_p) for i in range(P)])
        ctx = rd(ctx)
        if last:  # [CLS] rows only, fp32 residual (the fp16 stream's row widened)
            xres = res[cu[:-1]]
            if defect == "next_pair_residual":             # pair p reads the packed row of pair p + 1's [CLS]
                xres = np.concatenate([res[cu[1:-1]], np.zeros((1, H))])
            xc = _ln(ctx @ W(p + "wo").T + t[p + "bo"] + xres, t[p + "ln1_g"], t[p + "ln1_b"], eps)
            hdn = act(rd(xc) @ W(p + "w1").T + t[p + "b1"])
            xc = _ln(hdn @ W(p + "w2").T + t[p + "b2"] + xc, t[p + "ln2_g"], t[p + "ln2_b"], eps)
            break
        for (wn, bn, g, b) in ((None, None, "ln1_g", "ln1_b"), ("w1", "b1", "ln2_g", "ln2_b")):
            if wn is None:
                pre = ctx @ W(p + "wo").T + t[p + "bo"] + res
            else:
                pre = act(x16 @ W(p + wn).T + t[p + bn]) @ W(p + "w2").T + t[p + "b2"] + res
            if mode == "fp16":
                res = r16(_ln(r16(pre), t[p + g], t[p + b], eps))
            else:
                res = _ln(pre, t[p + g], t[p + b], eps)
            x16 = rd(res)
    pooled = np.tanh(xc @ t["pool_w"].T + t["pool_b"])
    return pooled @ t["cls_w"] + t["cls_b"][0], xc


# ------------------------------------------------------------------------------------------------ case table
def model_config(hidden, layers):
    return dict(vocab_size=VOCAB, hidden=hidden, layers=layers, heads=hidden // DH, intermediate=4 * hidden, max_pos=512,
                type_vocab=2, ln_eps=1e-12)


@functools.lru_cache(maxsize=3)
def model_weights(hidden, layers) -> CrossEncoderWeights:
    """N(0, sqrt(1.4 / H)) matrices, N(0, 0.1) biases and LayerNorm shifts, LayerNorm gains 1 + N(0, 0.1)."""
    w = CrossEncoderWeights.random(model_config(hidden, layers), seed=hidden + layers, std=math.sqrt(1.4 / hidden))
    rng = np.random.default_rng(1000 + hidden + layers)
    for name, a in w.tensors.items():
        base = name.split(".")[-1]
        if base.endswith("_g"):
            w.tensors[name] = (1.0 + 0.1 * rng.standard_normal(a.shape)).astype(np.float32)
        elif base.startswith("b") or base.endswith("_b"):
            w.tensors[name] = (0.1 * rng.standard_normal(a.shape)).astype(np.float32)
    return w


def straddle_lengths(S):
    """Lengths on both sides of every 16 / 32 / 64 / 128 / 256-key tile edge below S, then S - 1, S, 0 and S + 9
    (the last two clamp to 1 and S)."""
    edges = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257]
    out = []
    for n in [e for e in edges if e < S - 1] + [S - 1, S, 0, S + 9]:
        if n not in out:
            out.append(n)
    return out


@dataclass(frozen=True)
class Case:
    kind: str       # "rerank" (logits of ce_score) or "embed" (raw [CLS] state of enc_embed)
    hidden: int
    layers: int
    S: int

    @property
    def name(self):
        return f"{self.kind}-h{self.hidden}-l{self.layers}-s{self.S}"

    def weights(self):
        return model_weights(self.hidden, self.layers)


# S <= 128: mma<128, 2 or 3 heads per CTA>; 129..256: mma<256, 1>; 257..512: the generic kernel
WINDOWS = (32, 64, 128, 129, 200, 256, 257, 384, 512)
RERANK_CASES = ([Case("rerank", 128, 2, S) for S in WINDOWS] + [Case("rerank", 384, 2, S) for S in WINDOWS] +
                [Case("rerank", 256, 2, 128), Case("rerank", 256, 2, 300), Case("rerank", 768, 2, 128),
                 Case("rerank", 768, 2, 300), Case("rerank", 384, 6, 128)])
# one layer: only the [CLS] tail runs (no full-row attention); two layers: the full-row kernels, then the tail
EMBED_CASES = [Case("embed", H, L, S) for H in (128, 384, 768) for L in (1, 2) for S in (64, 300)]
CASES = RERANK_CASES + EMBED_CASES


def token_inputs(S, lengths, seed):
    """(input_ids, token_type, lengths) int32: random ids behind a [CLS], the second segment from a random split on;
    positions at or beyond a pair's length hold random ids too (the device must never read them)."""
    rng = np.random.default_rng(seed)
    lens = np.asarray(lengths, np.int32)
    P = len(lens)
    ids = rng.integers(0, VOCAB, (P, S)).astype(np.int32)
    ids[:, 0] = 101
    split = rng.integers(1, S + 1, P)
    tt = (np.arange(S)[None, :] >= split[:, None]).astype(np.int32)
    return ids, tt, lens


@functools.lru_cache(maxsize=None)
def case_inputs(case: Case):
    rng = np.random.default_rng(zlib.crc32(case.name.encode()))
    # three more random lengths where the CPU forward is cheap
    extra = [int(v) for v in rng.integers(1, case.S + 1, 3)] if case.S <= 128 else []
    return token_inputs(case.S, straddle_lengths(case.S) + extra, zlib.crc32(case.name.encode()) + 1)


@functools.lru_cache(maxsize=None)
def case_forward(case: Case, mode="fp64", defect=None):
    """The compared output of a case: logits (rerank) or [CLS] states (embed), for one mode / defect."""
    logits, cls = forward(case.weights(), *case_inputs(case), mode=mode, defect=defect)
    return logits if case.kind == "rerank" else cls


def case_streams(case: Case):
    """Residual streams the device runs the case on: the reranker both, the embedder fp32."""
    return ("fp16", "fp32") if case.kind == "rerank" else ("fp32",)


def case_tolerance(case: Case, stream: str) -> float:
    return tolerance(case_forward(case, stream), case_forward(case))
