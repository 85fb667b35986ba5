"""DPM-Solver++(2M) and (3M) SDE samplers for the v-parameterised ViewCrafter schedule (INTEGRATION.md "Samplers").

``DPMSolverSampler`` (two-way guidance, a ``ddim.DDIMSampler``) and ``DPMSolverSamplerMultiCond`` (three-way, a
``ddim_multiplecond.DDIMSampler``) take DDIM's ``sample()`` arguments and return its ``(samples, intermediates)``.  Each step is
DDIM's step with eta in {0, 1}, x_ddim, plus a multistep correction from the previous step's x0 prediction:

    x_prev = x_ddim + c (x0_i - x0_{i-1}),   c = sqrt(a') (1 - exp(-(1 + eta) h)) / (2 r),   r = h_{i-1} / h_i

with h the step in lambda = log(a / (1 - a)) / 2 (schedule.dpm_coefficients).  eta = 0 is DPM-Solver++(2M) (Lu et al. 2022,
Alg. 2), eta = 1 its SDE form, whose first-order part is DDIM with eta = 1.  The first step, a step after one that started at
a = 0 (zero terminal SNR) and the last step are first order: there c = 0 and the step is DDIM's, bit for bit.  The whole step is
one fused CUDA update (ops.dpm_update, vc_dpm_update); x0_i is taken before the dynamic rescale of pred_x0.

``DPMSolver3MSDESampler`` / ``DPMSolver3MSDESamplerMultiCond`` are the third-order multistep SDE solver (eta = 1 only), which keeps
the x0 of the two previous steps:

    x_prev = x_ddim + c1 (x0_i - x0_{i-1}) + c2 (x0_{i-1} - x0_{i-2})

(schedule.dpm3_coefficients; the phi2 d1 - phi3 d2 of k-diffusion's sample_dpmpp_3m_sde, written in differences).  Its first-order
steps are the 2M sampler's; where x0_{i-2} is not usable (c2 = 0) the step is the 2M step bit for bit.  One fused CUDA update
(ops.dpm3_update, vc_dpm3_update) reads both histories and writes x0_i over x0_{i-2}; the sampler then swaps the two buffers' roles.

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


def check_eta_sde(eta) -> float:
    eta = float(eta)
    if eta != 1.0:
        raise ValueError(f"DPM-Solver++(3M) SDE is defined for eta = 1 only, got eta={eta}")
    return eta


class _DPMSolverMixin:
    """What the DPM-Solver samplers add to their DDIM base class (first in the MRO).  A subclass names its solver, its eta check, its
    update (an ops function, looked up at call time), the keyword of each x0 history that update takes (most recent first) and the
    step-scalar key of each coefficient; make_schedule sets dpm_coefs, one float64 array of the coefficients per key."""
    solver_name = "DPM-Solver++(2M)"
    check_eta = staticmethod(check_eta)
    _op = "dpm_update"
    _hist_args = ("x0_hist",)
    _coef_keys = ("c_hist",)

    def _coefficients(self, ac, eta):
        return (schedule.dpm_coefficients(ac, self.ddim_timesteps, eta),)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        eta = self.check_eta(ddim_eta)
        super().make_schedule(ddim_num_steps, ddim_discretize, ddim_eta, verbose)
        ac = self.model.alphas_cumprod.detach().to("cpu", torch.float64).numpy()
        self.dpm_coefs = self._coefficients(ac, eta)

    @torch.no_grad()
    def sample(self, *args, **kwargs):
        """DDIMSampler.sample's arguments and return value.  eta must be one the solver defines (ValueError); mask, x0,
        noise_dropout > 0, temperature != 1, repeat_noise, timesteps, score_corrector and quantize_x0 raise NotImplementedError before
        any forward."""
        bound = inspect.signature(_ddim.DDIMSampler.sample).bind(self, *args, **kwargs).arguments
        given = dict(bound, **bound.get("kwargs", {}))
        for name, on in _UNSUPPORTED.items():
            if name in given and on(given[name]):
                raise NotImplementedError(f"{type(self).__name__}: sample({name}=...) is not supported by the {self.solver_name} sampler")
        self.check_eta(given.get("eta", 0.))
        self._x0_hist = None
        try:
            return super().sample(*args, **kwargs)
        finally:
            self._x0_hist = None

    def decode(self, *args, **kwargs):
        raise NotImplementedError(f"{type(self).__name__}.decode: the img2img helper is DDIM's; use ddim.DDIMSampler")

    def step_scalars(self, index: int, step: int) -> dict:
        d = super().step_scalars(index, step)
        for key, c in zip(self._coef_keys, self.dpm_coefs):
            d[key] = schedule.f32(c[index])
        return d

    def _fused_update(self, x, v_c, v_u, noise, sc, **extra):
        """DDIM's fused update with the solver's op.  The x0 histories (fp32, x's shape, most recent first) carry x0 from step to step
        and are sliced with the batch by the per-sample loop.  The op overwrites the oldest with this step's x0, which then becomes the
        most recent: the buffers rotate, nothing is copied."""
        hists = getattr(self, "_x0_hist", None)
        if hists is None or hists[0].shape != x.shape:
            if any(sc[k] != 0.0 for k in self._coef_keys):
                raise RuntimeError(f"{type(self).__name__}: a multistep step needs the previous steps' x0; call sample()")
            hists = [torch.empty(x.shape, device=x.device, dtype=torch.float32) for _ in self._hist_args]
        out = _ddim.DDIMSampler._fused_update(x, v_c, v_u, noise, sc, op=getattr(ops, self._op), **dict(zip(self._hist_args, hists)),
                                              **extra)
        self._x0_hist = hists[-1:] + hists[:-1]
        return out


class _DPMSolver3MSDEMixin(_DPMSolverMixin):
    """The third-order multistep SDE solver: two x0 histories, eta = 1."""
    solver_name = "DPM-Solver++(3M) SDE"
    check_eta = staticmethod(check_eta_sde)
    _op = "dpm3_update"
    _hist_args = ("x0_hist1", "x0_hist2")
    _coef_keys = ("c1", "c2")

    def _coefficients(self, ac, eta):
        return schedule.dpm3_coefficients(ac, self.ddim_timesteps)


class DPMSolverSampler(_DPMSolverMixin, _ddim.DDIMSampler):
    """DPM-Solver++(2M) with two-way guidance (the sampler of image_guided_synthesis(..., sampler="dpmpp_2m"))."""


class DPMSolverSamplerMultiCond(_DPMSolverMixin, _ddim_mc.DDIMSampler):
    """DPM-Solver++(2M) with three-way guidance (image_guided_synthesis(..., sampler="dpmpp_2m", multiple_cond_cfg=True))."""


class DPMSolver3MSDESampler(_DPMSolver3MSDEMixin, _ddim.DDIMSampler):
    """DPM-Solver++(3M) SDE with two-way guidance (the sampler of image_guided_synthesis(..., sampler="dpmpp_3m_sde"))."""


class DPMSolver3MSDESamplerMultiCond(_DPMSolver3MSDEMixin, _ddim_mc.DDIMSampler):
    """DPM-Solver++(3M) SDE with three-way guidance (image_guided_synthesis(..., sampler="dpmpp_3m_sde", multiple_cond_cfg=True))."""
