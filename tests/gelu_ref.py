"""The erf-GELU of the kernels, restated in numpy, and a per-element fp16 error bound for it.

Two device formulas compute gelu(x) = 0.5 x (1 + erf(x / sqrt 2)) with erf by Abramowitz-Stegun 7.1.26,
    erf(z) ~ 1 - p(t) t exp(-z^2),   t = 1 / (1 + 0.3275911 |z|),   p a degree-4 polynomial,
in fp32, and round the result to fp16 once:
  * "fast": `gelu_erf_fast` of viewcrafter_b200/csrc/common.cuh (ops.gelu_f16): t = __frcp_rn(fma(..)), e = __expf(-z^2)
    (ex2.approx of the argument times log2 e), y = 1 - (p t) e, then 0.5 x (1 + copysign(y, z));
  * "epilogue": `gelu_epilogue` of gemm_common.cuh (the GEGLU epilogue of the tap-GEMM): t = rcp.approx, e = ex2.approx, erf_abs =
    fma(-(p t), e, 1), then fma(0.5 x, copysign(erf_abs, z), 0.5 x).
`gelu_model` restates either with exact exp and exactly rounded reciprocals (the approximate MUFU results are covered by the bound).

`gelu_bound(x)` bounds |fp16 kernel output - gelu(x)| element by element.  u = 2^-24 is the fp32 unit roundoff; every term is a
worst case over the operations it names, with z = x / sqrt 2, e = exp(-z^2), and P = sum |a_k| t^k, P' = sum k |a_k| t^k over the five
A&S coefficients a_k (so |p(t) t| <= P and |t d(p(t) t)/dt| <= P'):
  (a) the A&S formula itself: |erf_AS(z) - erf(z)| <= 1.5e-7 for every z (A&S 7.1.26);
  (b) the reciprocal: fma(0.3275911, |z|, 1) rounds once (u) and rcp.approx is within 1 ulp (2u), so t is within 4u relative (with
      margin); a relative error d in t moves p(t) t by at most P' d, and the product by e;
  (c) Horner: four fma and one multiply (p t), each rounding once, perturb p(t) t by at most gamma_10 P <= 10.1 u P, times e;
  (d) the exponential: -z^2 and its product with log2 e round twice (the constant log2 e once more), so the exp2 argument is within 3u
      relative and exp moves by z^2 3u relative; ex2.approx is within 2 ulp (4u) relative; both times P.  ex2.approx.ftz flushes
      results below 2^-126 to zero: 2^-126 P more;
  (e) the cancellation: y = 1 - p t e rounds to fp32 (u |y|), and 1 + y rounds again in the fast path (u (1 + erf)); the epilogue's
      fma rounds 0.5 x (1 + erf) once, which (f) covers;
  (f) the argument: z = fl(x * fl(1/sqrt 2)) is within 2u relative, and erf moves by (2/sqrt pi) e |z| 2u;
  (g) the last fp32 product (fast: 0.5 x times 1 + erf; epilogue: the fma) rounds once: u |gelu(x)|, doubled for margin.
err = 0.5 |x| ((a) + (b) + (c) + (d) + (e) + (f)) + (g) is the fp32 error; the fp16 store adds half an fp16 ulp of a value within
err of the exact one, so  bound = err + half_ulp_fp16(|gelu(x)| + err)  (fp16 subnormal spacing below 2^-14).

None of it is fitted to a GPU run.  Where gelu(x) is tiny (the negative tail), term (a) is several fp16 subnormal ulps: the kernels
are not within half an ulp there, and no fp32 A&S evaluation can be.
"""
import math

import numpy as np
from scipy.special import erfc

F32 = np.float32
U = 2.0 ** -24
AS_ERR = 1.5e-7
AS_P = 0.3275911
AS_A = (0.254829592, -0.284496736, 1.421413741, -1.453152027, 1.061405429)     # a_1 .. a_5 of p(t) t = sum a_k t^k
INV_SQRT2 = 0.70710678118654752440
LOG2E = 1.4426950408889634


def finite_fp16() -> np.ndarray:
    """Every finite fp16 value (63,488 of them, -0 included), in bit-pattern order."""
    h = np.arange(1 << 16, dtype=np.uint16).view(np.float16)
    return h[np.isfinite(h)]


def gelu_ref(x) -> np.ndarray:
    """float64 0.5 x (1 + erf(x / sqrt 2)), written with erfc so that the negative tail does not cancel."""
    xd = np.asarray(x, dtype=np.float64)
    return 0.5 * xd * erfc(-xd / math.sqrt(2.0))


def _fma(a, b, c):
    # an fp32 fma: the fp32 x fp32 product is exact in float64, the sum rounds once in float64 and once more to fp32 (a 2^-53 slip)
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def gelu_model(x, path="fast", mutant=None, f32=False):
    """fp16 gelu of fp16 inputs as the kernels compute it (module docstring); f32: the fp32 value before the fp16 store.  mutant: "tanh" (the tanh approximation), "sigmoid"
    (x sigmoid(1.702 x)), "no-rsqrt2" (erf(x) instead of erf(x / sqrt 2)), "no-half" (the 0.5 dropped)."""
    x = np.asarray(x, np.float16).astype(F32)
    with np.errstate(all="ignore"):
        if mutant == "tanh":
            xd = x.astype(np.float64)
            g = (0.5 * xd * (1 + np.tanh(math.sqrt(2 / math.pi) * (xd + 0.044715 * xd ** 3)))).astype(F32)
            return g if f32 else g.astype(np.float16)
        if mutant == "sigmoid":
            g = (x / (F32(1) + np.exp(F32(-1.702) * x))).astype(F32)
            return g if f32 else g.astype(np.float16)
        z = x if mutant == "no-rsqrt2" else (x * F32(INV_SQRT2)).astype(F32)
        az = np.abs(z)
        t = (1.0 / _fma(F32(AS_P), az, F32(1)).astype(np.float64)).astype(F32)
        p = _fma(F32(AS_A[4]), t, F32(AS_A[3]))
        for a in AS_A[2::-1]:
            p = _fma(p, t, F32(a))
        pt = (p * t).astype(F32)
        if path == "fast":
            arg = ((-az * az).astype(F32) * F32(LOG2E)).astype(F32)
            e = np.exp2(arg.astype(np.float64)).astype(F32)
            y = _fma(-pt, e, F32(1))
            one_p = (F32(1) + np.copysign(y, z)).astype(F32)
            g = ((F32(0.5) if mutant != "no-half" else F32(1)) * x * one_p).astype(F32)
        else:
            arg = ((az * az).astype(F32) * F32(-LOG2E)).astype(F32)
            e = np.exp2(arg.astype(np.float64)).astype(F32)
            erf_abs = _fma(-pt, e, F32(1))
            hx = (F32(0.5) if mutant != "no-half" else F32(1)) * x
            g = _fma(hx, np.copysign(erf_abs, z), hx)
        return g if f32 else g.astype(np.float16)


def gelu_bound(x) -> np.ndarray:
    """float64 bound on |fp16 gelu - gelu(x)| per element (module docstring); finite x only."""
    return fp32_error_bound(x) + half_ulp_fp16(np.abs(gelu_ref(x)) + fp32_error_bound(x))


def fp32_error_bound(x) -> np.ndarray:
    """err of the module docstring, terms (a)-(g): the bound on the fp32 value before the fp16 store."""
    xd = np.asarray(x, np.float16).astype(np.float64)
    assert np.all(np.isfinite(xd))
    ref = gelu_ref(xd)
    z = np.abs(xd) * INV_SQRT2
    with np.errstate(under="ignore"):
        e = np.exp(-z * z)
    t = 1.0 / (1.0 + AS_P * z)
    P = sum(abs(a) * t ** (k + 1) for k, a in enumerate(AS_A))
    Pd = sum((k + 1) * abs(a) * t ** (k + 1) for k, a in enumerate(AS_A))
    y = 1.0 - P * e
    one_p_erf = np.abs(2.0 * ref / np.where(xd == 0, 1.0, xd))         # 1 + erf(x / sqrt 2)
    D = (AS_ERR                                                       # (a)
         + e * Pd * 4 * U                                              # (b)
         + e * P * 10.1 * U                                            # (c)
         + e * P * (3 * U * z * z + 4 * U) + 2.0 ** -126 * P           # (d)
         + U * np.abs(y) + U * one_p_erf                               # (e)
         + (2 / math.sqrt(math.pi)) * e * z * 2 * U)                   # (f)
    return 0.5 * np.abs(xd) * D + 2 * U * np.abs(ref)                # (g)


def half_ulp_fp16(v) -> np.ndarray:
    """Half the fp16 spacing at |v| (v >= 0, float64), 16 from 32768 up to the largest finite fp16 value."""
    v = np.asarray(v, np.float64)
    small = np.minimum(v, 32752.0).astype(np.float16)
    return np.where(v >= 32768.0, 16.0, 0.5 * np.spacing(small).astype(np.float64))


def worst_ratio(out16, x) -> tuple:
    """(max |out - gelu(x)| / bound, the x where it is reached) over finite x; out is fp16 (or the fp32 value before the store:
    then pass fp32_error_bound's share by dividing yourself).  A non-finite output counts as an infinite ratio."""
    with np.errstate(invalid="ignore"):
        r = np.abs(np.asarray(out16).astype(np.float64) - gelu_ref(x)) / gelu_bound(x)
    r = np.where(np.isnan(r), np.inf, r)
    k = int(np.argmax(r))
    return float(r[k]), float(np.asarray(x, np.float16)[k])
