"""DPM-Solver++(2M) samplers for the v-parameterised ViewCrafter schedule (INTEGRATION.md "Samplers").

``DPMSolverSampler`` (two-way guidance, a ``ddim.DDIMSampler``) and ``DPMSolverSamplerMultiCond`` (three-way, a
``ddim_multiplecond.DDIMSampler``) take DDIM's ``sample()`` arguments and return its ``(samples, intermediates)``.  Each step is
DDIM's step with eta in {0, 1}, x_ddim, plus a multistep correction from the previous step's x0 prediction:

    x_prev = x_ddim + c (x0_i - x0_{i-1}),   c = sqrt(a') (1 - exp(-(1 + eta) h)) / (2 r),   r = h_{i-1} / h_i

with h the step in lambda = log(a / (1 - a)) / 2 (schedule.dpm_coefficients).  eta = 0 is DPM-Solver++(2M) (Lu et al. 2022,
Alg. 2), eta = 1 its SDE form, whose first-order part is DDIM with eta = 1.  The first step, a step after one that started at
a = 0 (zero terminal SNR) and the last step are first order: there c = 0 and the step is DDIM's, bit for bit.  The whole step is
one fused CUDA update (ops.dpm_update, vc_dpm_update); x0_i is taken before the dynamic rescale of pred_x0.

Everything else is inherited: CFG batching, the shared prefix, the three-way forwards, the multi-GPU CFG split, the per-sample
update at B > 1 with guidance rescale, each class's ddim_scale_arr_prev, and the random numbers -- x_T and one noise tensor per
step, also at eta = 0 where the noise is multiplied by 0, so the generator advances exactly as under DDIMSampler.sample and
skip_sample_draws / replica groups work unchanged.
"""
from __future__ import annotations

import inspect

import torch

from . import ops, schedule
from . import ddim as _ddim
from . import ddim_multiplecond as _ddim_mc

# sample() options the multistep update does not define: name -> test of the value that turns the option on
_UNSUPPORTED = {"mask": lambda v: v is not None, "x0": lambda v: v is not None, "noise_dropout": lambda v: v > 0.,
                "temperature": lambda v: v != 1., "repeat_noise": bool, "timesteps": lambda v: v is not None,
                "score_corrector": lambda v: v is not None, "quantize_x0": bool}


def check_eta(eta) -> float:
    eta = float(eta)
    if eta not in (0.0, 1.0):
        raise ValueError(f"DPM-Solver++(2M) is defined for eta = 0 (ODE) and eta = 1 (SDE), got eta={eta}")
    return eta


class _DPMSolverMixin:
    """What the two DPM-Solver samplers add to their DDIM base class (first in the MRO)."""

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        eta = check_eta(ddim_eta)
        super().make_schedule(ddim_num_steps, ddim_discretize, ddim_eta, verbose)
        ac = self.model.alphas_cumprod.detach().to("cpu", torch.float64).numpy()
        self.dpm_c_hist = schedule.dpm_coefficients(ac, self.ddim_timesteps, eta)

    @torch.no_grad()
    def sample(self, *args, **kwargs):
        """DDIMSampler.sample's arguments and return value.  eta must be 0 or 1 (ValueError); mask, x0, noise_dropout > 0,
        temperature != 1, repeat_noise, timesteps, score_corrector and quantize_x0 raise NotImplementedError before any forward."""
        bound = inspect.signature(_ddim.DDIMSampler.sample).bind(self, *args, **kwargs).arguments
        given = dict(bound, **bound.get("kwargs", {}))
        for name, on in _UNSUPPORTED.items():
            if name in given and on(given[name]):
                raise NotImplementedError(f"{type(self).__name__}: sample({name}=...) is not supported by the DPM-Solver++(2M) sampler")
        check_eta(given.get("eta", 0.))
        self._x0_hist = None
        try:
            return super().sample(*args, **kwargs)
        finally:
            self._x0_hist = None

    def decode(self, *args, **kwargs):
        raise NotImplementedError(f"{type(self).__name__}.decode: the img2img helper is DDIM's; use ddim.DDIMSampler")

    def step_scalars(self, index: int, step: int) -> dict:
        d = super().step_scalars(index, step)
        d["c_hist"] = schedule.f32(self.dpm_c_hist[index])
        return d

    def _fused_update(self, x, v_c, v_u, noise, sc, **extra):
        """DDIM's fused update with ops.dpm_update; x0_hist (fp32, x's shape) carries x0 from step to step and is sliced with the
        batch by the per-sample loop."""
        hist = getattr(self, "_x0_hist", None)
        if hist is None or hist.shape != x.shape:
            if sc["c_hist"] != 0.0:
                raise RuntimeError(f"{type(self).__name__}: a second-order step needs the previous step's x0; call sample()")
            hist = self._x0_hist = torch.empty(x.shape, device=x.device, dtype=torch.float32)
        return _ddim.DDIMSampler._fused_update(x, v_c, v_u, noise, sc, op=ops.dpm_update, x0_hist=hist, **extra)


class DPMSolverSampler(_DPMSolverMixin, _ddim.DDIMSampler):
    """DPM-Solver++(2M) with two-way guidance (the sampler of image_guided_synthesis(..., sampler="dpmpp_2m"))."""


class DPMSolverSamplerMultiCond(_DPMSolverMixin, _ddim_mc.DDIMSampler):
    """DPM-Solver++(2M) with three-way guidance (image_guided_synthesis(..., sampler="dpmpp_2m", multiple_cond_cfg=True))."""
