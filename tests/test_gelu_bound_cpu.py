"""The erf-GELU bound of `tests/gelu_ref.py` holds for the kernels' arithmetic on every finite fp16 input and is tight enough to catch
the usual wrong GELUs.

`gelu_model` restates `gelu_erf_fast` (ops.gelu_f16) and `gelu_epilogue` (the GEGLU epilogue) in numpy fp32.  On all 63,488 finite fp16
inputs both must stay within the bound after the fp16 store, and their fp32 values within 0.8 of the bound's fp32 share (the A&S
formula error alone reaches about 0.7 of it).  Each mutant must break the bound.
"""
import numpy as np
import pytest

from tests import gelu_ref as G


def _fp32_share(path):
    x = G.finite_fp16()
    d = np.abs(G.gelu_model(x, path, f32=True).astype(np.float64) - G.gelu_ref(x))
    eb = G.fp32_error_bound(x)
    assert np.all((eb > 0) | (d == 0))                     # x = 0 only: exact
    r = np.where(eb > 0, d / np.where(eb > 0, eb, 1.0), 0.0)
    k = int(np.argmax(r))
    return float(r[k]), float(x[k])


@pytest.mark.parametrize("path", ["fast", "epilogue"])
def test_model_within_the_bound_on_every_fp16_input(path):
    x = G.finite_fp16()
    assert x.size == 63488
    r16, x16 = G.worst_ratio(G.gelu_model(x, path), x)
    r32, x32 = _fp32_share(path)
    ref = G.gelu_ref(x)
    ulps = np.abs(G.gelu_model(x, path).astype(np.float64) - ref.astype(np.float16).astype(np.float64)) / (2 * G.half_ulp_fp16(np.abs(ref)))
    print(f"{path}: fp16 error / bound {r16:.4f} at x={x16:.5g}; fp32 error / fp32 share {r32:.4f} at x={x32:.5g}; "
          f"{float(ulps.max()):.0f} fp16 ulps from the rounded reference at most")
    assert r16 <= 1.0 and r32 <= 0.8


@pytest.mark.parametrize("mutant", ["tanh", "sigmoid", "no-rsqrt2", "no-half"])
def test_mutant_breaks_the_bound(mutant):
    x = G.finite_fp16()
    r, at = G.worst_ratio(G.gelu_model(x, "fast", mutant), x)
    print(f"{mutant}: error / bound {r:.4g} at x={at:.5g}")
    assert r > 1.0, f"{mutant} stays within the bound ({r:.3g})"

