"""CPU checks of the cross-encoder numerics (tests/ce_numerics.py) that the GPU parity tests rely on:

* the fp64 forward is ``oracle.cross_encoder.numpy_forward`` (itself pinned to HuggingFace) on the device's clamped
  lengths;
* the device-rounding emulation stays in the band of its fp64 distance that the weights predict;
* power: at the case table's weights every seeded attention / [CLS]-tail defect moves the fp64 output by at least 5 x
  the case's tolerance, so a GPU test at that tolerance would fail on it.
"""
import math

import numpy as np
import pytest

import ce_numerics as cn
from oracle.cross_encoder import _gelu, numpy_forward


@pytest.mark.parametrize("hidden,layers,S", [(128, 2, 64), (384, 1, 128), (256, 2, 160)])
def test_fp64_forward_equals_numpy_oracle(hidden, layers, S):
    w = cn.model_weights(hidden, layers)
    lens = cn.straddle_lengths(S)
    ids, tt, lens = cn.token_inputs(S, lens, seed=S)
    logits, cls = cn.forward(w, ids, tt, lens)
    # numpy_forward attends over all S padded keys when len = 0; the device (and forward) clamp to [1, S]
    want, _ = numpy_forward(w, ids, tt, np.clip(lens, 1, S))
    assert np.allclose(logits, want, rtol=1e-10, atol=1e-12), np.abs(logits - want).max()
    assert cls.shape == (len(lens), hidden)
    # len 0 and len > S are the same pairs as len 1 and len S
    i0, iS = list(lens).index(0), list(lens).index(S + 9)
    same = cn.forward(w, ids[[i0, iS]], tt[[i0, iS]], [1, S])[0]
    assert np.allclose(same, logits[[i0, iS]], rtol=1e-12, atol=1e-12)


def test_packed_half_gelu_tracks_the_erf_gelu():
    x = cn.r16(np.linspace(-8.0, 8.0, 200001))
    err = np.abs(cn.gelu_fp16(x) - _gelu(x))
    # every step rounds to fp16: up to 1.3e-3 near |x| = 3 where the result's ulp is 2e-3, rms 2.4e-4
    # (scripts/fit_gelu.py: 2.0e-4 rms on N(0, 1) inputs)
    assert err.max() <= 2e-3 and np.sqrt(np.mean(err ** 2)) <= 4e-4, (err.max(), np.sqrt(np.mean(err ** 2)))


@pytest.mark.parametrize("case", cn.CASES, ids=lambda c: c.name)
def test_emulation_stays_in_the_predicted_band(case):
    """At std sqrt(1.4 / H) the fp16 GEMM operands move logits and [CLS] elements by ~1e-3 (both residual streams):
    an emulation much closer to fp64 rounds nothing, one much further rounds the wrong thing."""
    ref = cn.case_forward(case)
    for stream in cn.case_streams(case):
        err = float(np.max(np.abs(cn.case_forward(case, stream) - ref)))
        assert 1e-4 <= err <= 5e-3, (case.name, stream, err)


@pytest.mark.parametrize("case", cn.CASES, ids=lambda c: c.name)
def test_every_defect_moves_the_output_5x_past_the_tolerance(case):
    ref = cn.case_forward(case)
    tol = max(cn.case_tolerance(case, s) for s in cn.case_streams(case))
    for defect in cn.DEFECTS:
        moved = float(np.max(np.abs(cn.case_forward(case, "fp64", defect) - ref)))
        assert moved >= 5.0 * tol, (case.name, defect, moved, tol)


def test_case_table_covers_every_attention_kernel_and_model_shape():
    windows = {c.S for c in cn.RERANK_CASES}
    assert {32, 64, 128} <= windows and {129, 200, 256} <= windows and {257, 384, 512} <= windows
    assert {c.hidden for c in cn.RERANK_CASES} == {128, 256, 384, 768}
    assert any(c.layers == 6 for c in cn.RERANK_CASES)
    assert {(c.hidden, c.layers, c.S) for c in cn.EMBED_CASES} == {(h, l, s) for h in (128, 384, 768) for l in (1, 2)
                                                                   for s in (64, 300)}
    for c in cn.CASES:
        w = c.weights()
        assert math.isclose(float(np.std(w.tensors["l0.wq"])), math.sqrt(1.4 / c.hidden), rel_tol=0.02)
        assert np.any(w.tensors["l0.bq"] != 0) and np.any(w.tensors["l0.ln1_g"] != 1)
        lens = cn.case_inputs(c)[2]
        assert 0 in lens and lens.max() > c.S and (c.S - 1) in lens
        assert all(n in lens for n in (1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257) if n < c.S)
