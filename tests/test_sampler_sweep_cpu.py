"""Where the eta = 1 DDIM radicand 1 - a' - sigma^2 rounds below zero, and the step counts the GPU sampler sweep
(tests/test_sampler_sweep_gpu.py) runs its guidance grid and end-to-end samples at.

At eta = 1 the first uniform_trailing step starts from a = 0 (zero terminal SNR), where 1 - a' - sigma^2 is 0 in exact arithmetic.  The
update kernels evaluate it from the fp32 step scalars as FADD (1 - a') then FFMA (- sigma sigma + that) -- one rounding fewer than the
reference's unfused torch expression ``1.0 - a_prev - sigma_t ** 2`` -- and either can come out below zero.  `radicands` recomputes both
from the samplers' own step_scalars; the test pins which step counts go negative, so that the sweep's chosen step counts keep covering
the edge.
"""
import numpy as np
import torch

from viewcrafter_b200 import schedule
from viewcrafter_b200.ddim import DDIMSampler

SPACINGS = ("uniform_trailing", "uniform")
BASE_SCALES = (0.3, 0.7)
MAX_STEPS = 100
CFG_STEPS = (4, 7, 9, 25, 50)         # the full guidance grid: fused radicand < 0 with the reference's >= 0 (4, 9), both < 0 (7, 25), >= 0 (50)
E2E_STEPS = (4, 25)                   # DDIM samplers end to end at eta = 1


class ScheduleModel:
    """The schedule buffers DDIMSampler.make_schedule reads, with dynamic rescale on (LatentDiffusion's defaults)."""
    parameterization = "v"
    use_dynamic_rescale = True
    num_timesteps = 1000

    def __init__(self, base_scale):
        for k, v in schedule.model_buffers(base_scale=base_scale).items():
            setattr(self, k, v)


def step_counts(spacing):
    """S in 1..MAX_STEPS whose timesteps lie in 0..999.  "uniform" reaches t = 1000 at S = 3, 9, 27, 36 and 37, where DDIM's tables
    fail (the reference's too, see test_dpm_solver_cpu.py); "uniform_trailing" at S = 61 gets a 62nd timestep, t = -1, from the float
    arange, which wraps to t = 999 and gives sigma = NaN in the reference's tables and in the sampler's alike."""
    ok = lambda ts: ts.min() >= 0 and ts.max() < 1000
    return [S for S in range(1, MAX_STEPS + 1) if ok(schedule.ddim_timesteps(spacing, S, 1000))]


def sampler_steps(sampler, spacing, S, eta):
    """[(index, step_scalars)] of one sample() call of `sampler` (a DDIM or DPM-Solver sampler on a ScheduleModel), in sampling order."""
    sampler.make_schedule(S, spacing, eta, verbose=False)
    ts = sampler.ddim_timesteps
    return [(j, sampler.step_scalars(j, int(ts[j]))) for j in range(len(ts) - 1, -1, -1)]


def radicands(spacing, S, eta):
    """{index: (fused, unfused)} fp32 values of 1 - a' - sigma^2 of each step: the kernels' FADD + FFMA, and the reference's torch
    expression (three roundings)."""
    out = {}
    for j, sc in sampler_steps(DDIMSampler(ScheduleModel(0.3)), spacing, S, eta):
        ap, sg = np.float32(sc["a_prev"]), np.float32(sc["sigma_t"])
        r = np.float32(1.0) - ap
        fused = np.float32(np.float64(r) - np.float64(sg) * np.float64(sg))      # the fp32 product is exact in float64
        a_t, s_t = torch.tensor(sc["a_prev"], dtype=torch.float32), torch.tensor(sc["sigma_t"], dtype=torch.float32)
        unfused = float(1.0 - a_t - s_t ** 2)
        out[j] = (float(fused), unfused)
    return out


def negative_radicands(spacing, eta):
    """(fused, unfused): sorted step counts S with a step whose radicand is < 0."""
    fused, unfused = set(), set()
    for S in step_counts(spacing):
        for j, (f, u) in radicands(spacing, S, eta).items():
            if f < 0:
                fused.add(S)
            if u < 0:
                unfused.add(S)
    return sorted(fused), sorted(unfused)


def test_negative_radicands_are_in_the_swept_step_counts():
    fused, unfused = negative_radicands("uniform_trailing", 1.0)
    print(f"uniform_trailing, eta = 1: fused fp32 radicand < 0 at S = {fused}")
    print(f"uniform_trailing, eta = 1: the reference's unfused fp32 radicand < 0 at S = {unfused}")
    only_fused = sorted(set(fused) - set(unfused))
    print(f"fused < 0 where the reference's is >= 0 (the library returned NaN, the reference a sample): S = {only_fused}")
    # only the first step (index S - 1, from a = 0) has an exact radicand of 0; every radicand is a number
    for S in step_counts("uniform_trailing"):
        r = radicands("uniform_trailing", S, 1.0)
        assert len(r) == S and all(np.isfinite(v) for fu in r.values() for v in fu), S
        assert all(f >= 0 and u >= 0 for j, (f, u) in r.items() if j != S - 1), S
    assert len(fused) > 30 and set(fused) <= set(step_counts("uniform_trailing"))
    # the guidance grid and the end-to-end runs sit on both sides of the edge
    assert {4, 9} <= set(CFG_STEPS) & set(only_fused)
    assert set(CFG_STEPS) & set(fused) & set(unfused) and set(CFG_STEPS) - set(fused)
    assert set(E2E_STEPS) <= set(fused) and 4 not in unfused           # S = 4 is compared with the reference's loop
    for spacing, eta in (("uniform_trailing", 0.0), ("uniform", 0.0), ("uniform", 1.0)):
        assert negative_radicands(spacing, eta) == ([], []), (spacing, eta)
