"""Host-side (numpy, float64 -> float32) diffusion schedule tables.  Bit-exactness against the reference is
checked by tests/test_schedule_cpu.py using known answers generated from the reference's own functions.

Mirrors: make_beta_schedule / rescale_zero_terminal_snr / make_ddim_timesteps / make_ddim_sampling_parameters
(lvdm/models/utils_diffusion.py:31-91,112-144), DDPM.register_schedule (lvdm/models/ddpm3d.py:123-150),
LatentDiffusion scale_arr (ddpm3d.py:522-527) and DDIMSampler.make_schedule (lvdm/models/samplers/ddim.py:24-59).
"""
from __future__ import annotations

import numpy as np
import torch


def linear_betas(n: int, start: float, end: float) -> np.ndarray:
    return (torch.linspace(start ** 0.5, end ** 0.5, n, dtype=torch.float64, device="cpu") ** 2).numpy()


def zero_terminal_snr(betas: np.ndarray) -> np.ndarray:
    root = np.sqrt(np.cumprod(1.0 - betas, axis=0))
    r0, rT = root[0].copy(), root[-1].copy()
    root = (root - rT) * (r0 / (r0 - rT))
    bar = root ** 2
    return 1 - np.concatenate([bar[0:1], bar[1:] / bar[:-1]])


def model_buffers(timesteps=1000, linear_start=0.00085, linear_end=0.012, zero_snr=True, base_scale=0.3,
                  turning_step=400, dynamic_rescale=True) -> dict:
    betas = linear_betas(timesteps, linear_start, linear_end)
    if zero_snr:
        betas = zero_terminal_snr(betas)
    ac = np.cumprod(1.0 - betas, axis=0)
    t32 = lambda a: torch.tensor(a, dtype=torch.float32, device="cpu")
    out = dict(betas=t32(betas), alphas_cumprod=t32(ac), alphas_cumprod_prev=t32(np.append(1.0, ac[:-1])),
               sqrt_alphas_cumprod=t32(np.sqrt(ac)), sqrt_one_minus_alphas_cumprod=t32(np.sqrt(1.0 - ac)))
    if dynamic_rescale:
        out["scale_arr"] = t32(np.concatenate((np.linspace(1.0, base_scale, turning_step), np.full(timesteps, base_scale))))
    return out


def ddim_timesteps(method: str, n_ddim: int, n_ddpm: int) -> np.ndarray:
    if method == "uniform":
        return np.asarray(list(range(0, n_ddpm, n_ddpm // n_ddim))) + 1
    if method == "uniform_trailing":
        return np.flip(np.round(np.arange(n_ddpm, 0, -(n_ddpm / n_ddim)))).astype(np.int64) - 1
    if method == "quad":
        return ((np.linspace(0, np.sqrt(n_ddpm * .8), n_ddim)) ** 2).astype(int) + 1
    raise NotImplementedError(f'There is no ddim discretization method called "{method}"')


def ddim_parameters(alphacums: torch.Tensor, ts: np.ndarray, eta: float):
    """Returns (sigmas float64 tensor, alphas float32 tensor, alphas_prev float64 ndarray): the reference's dtypes."""
    alphas = alphacums[ts]
    alphas_prev = np.asarray([alphacums[0]] + alphacums[ts[:-1]].tolist())
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    return sigmas, alphas, alphas_prev


def dpm_coefficients(alphacums, ts: np.ndarray, eta: float) -> np.ndarray:
    """float64 [S]: c of the DPM-Solver++(2M) step of DDIM index j (INTEGRATION.md "Samplers"), which goes from a = alphacums[ts[j]] to
    a' = alphacums[ts[j - 1]] (alphacums[0] for j = 0) with h_j = lambda(a') - lambda(a), lambda = log(a / (1 - a)) / 2:
        c_j = sqrt(a') (1 - exp(-(1 + eta) h_j)) / (2 r),   r = h_{j+1} / h_j   (step j + 1 is the one sampled before step j).
    c_j = 0 -- a first-order (DDIM) step -- on the first step (j = S - 1), the last (j = 0), after a step that started at a = 0
    (h_{j+1} infinite) and where h_j or h_{j+1} is 0 (repeated timesteps of the "quad" spacing)."""
    ac = np.asarray(alphacums, dtype=np.float64)
    a = ac[ts]
    a_prev = np.concatenate([ac[0:1], a[:-1]])
    with np.errstate(divide="ignore"):
        lam = lambda v: 0.5 * (np.log(v) - np.log1p(-v))
        h = lam(a_prev) - lam(a)
    c = np.zeros(len(ts), dtype=np.float64)
    for j in range(1, len(ts) - 1):
        if np.isfinite(h[j + 1]) and h[j + 1] != 0 and h[j] != 0:
            c[j] = np.sqrt(a_prev[j]) * -np.expm1(-(1.0 + eta) * h[j]) * h[j] / (2.0 * h[j + 1])
    return c


def dpm3_coefficients(alphacums, ts: np.ndarray):
    """float64 ([S], [S]): (c1, c2) of the DPM-Solver++(3M) SDE step (eta = 1) of DDIM index j (INTEGRATION.md "Samplers"), with a, a',
    lambda and h_j as in dpm_coefficients, h_e = 2 h_j, r0 = h_{j+1} / h_j and r1 = h_{j+2} / h_j:
        phi2 = expm1(-h_e) / h_e + 1,   phi3 = phi2 / h_e - 1/2
        c1_j = sqrt(a') [phi2 (1 + r0 / (r0 + r1)) - phi3 / (r0 + r1)] / r0,   c2_j = sqrt(a') [phi3 / (r0 + r1) - phi2 r0 / (r0 + r1)] / r1
    Fallbacks: c1 = c2 = 0 (first order) wherever dpm_coefficients(..., eta=1) is 0; otherwise, where h_{j+2} is infinite (step j + 2
    started at a = 0), zero or absent (j + 2 = S), c2 = 0 and c1 is dpm_coefficients' c exactly (the 2M step)."""
    ac = np.asarray(alphacums, dtype=np.float64)
    a = ac[ts]
    a_prev = np.concatenate([ac[0:1], a[:-1]])
    with np.errstate(divide="ignore"):
        lam = lambda v: 0.5 * (np.log(v) - np.log1p(-v))
        h = lam(a_prev) - lam(a)
    c1 = dpm_coefficients(ac, ts, 1.0)
    c2 = np.zeros(len(ts), dtype=np.float64)
    for j in range(1, len(ts) - 2):
        if c1[j] != 0 and np.isfinite(h[j + 2]) and h[j + 2] != 0:
            he = 2.0 * h[j]
            r0, r1 = h[j + 1] / h[j], h[j + 2] / h[j]
            phi2 = np.expm1(-he) / he + 1.0
            phi3 = phi2 / he - 0.5
            c1[j] = np.sqrt(a_prev[j]) * (phi2 * (1.0 + r0 / (r0 + r1)) - phi3 / (r0 + r1)) / r0
            c2[j] = np.sqrt(a_prev[j]) * (phi3 / (r0 + r1) - phi2 * r0 / (r0 + r1)) / r1
    return c1, c2


def f32(v) -> float:
    """The value torch.full(size, v) would hold (float32 rounding of a python/numpy/tensor scalar)."""
    return float(np.float32(float(v)))
