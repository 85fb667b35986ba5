"""Drop-in ``DDIMSampler`` with three-way classifier-free guidance (reference: lvdm/models/samplers/ddim_multiplecond.py),
the sampler ``image_guided_synthesis(..., multiple_cond_cfg=True)`` selects (utils/diffusion_utils.py:9,119).

Differences from ``viewcrafter_b200.ddim.DDIMSampler`` -- exactly the reference's:
  * three ``apply_model`` calls per step: cond, uncond and ``unconditional_conditioning_img_nonetext`` (image kept, text
    dropped), combined as ``u + cfg_img (v_img - u) + s (v_cond - v_img)`` (ddim_multiplecond.py:227-233);
    ``cfg_img`` defaults to the text scale;
  * ``ddim_scale_arr_prev[0] = ddim_scale_arr[0]`` (ddim_multiplecond.py:33; ddim.py:33-35 fixed this one only), so the last
    step's dynamic rescale differs between the two samplers (SURVEY.md App. D).
The combine, guidance rescale, v->(eps, x0), dynamic rescale and x_{t-1} are one fused CUDA update (vc_ddim_update3).

How the three predictions are computed (none of it draws random numbers, so the RNG stream is the reference's):
  * ``batch_cfg=True`` and stackable conditioning (dicts with equal keys): ONE B=3 forward of (cond, uncond, uncond_img),
    which computes the context-free prefix once when the c_concat entries are shared; otherwise B=2 (cond, uncond) + B=1;
  * ``batch_cfg=False``: three forwards, like the reference;
  * multi-GPU 2-way CFG split (parallel.shard_model(cfg_split=True)): the first half of the ranks computes cond (B=1), the
    second half uncond and uncond_img (one B=2 forward when stackable), and the pairs swap their predictions.
"""
from __future__ import annotations

import torch

from . import ops
from .ddim import DDIMSampler as _TwoWaySampler


class DDIMSampler(_TwoWaySampler):
    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        super().make_schedule(ddim_num_steps, ddim_discretize, ddim_eta, verbose)
        if self.use_dynamic_rescale:
            self.ddim_scale_arr_prev = torch.cat([self.ddim_scale_arr[0:1], self.ddim_scale_arr[:-1]])

    @torch.no_grad()
    def p_sample_ddim(self, x, c, t, index, repeat_noise=False, use_original_steps=False, quantize_denoised=False,
                      temperature=1., noise_dropout=0., score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1., unconditional_conditioning=None, uc_type=None, cfg_img=None,
                      mask=None, x0=None, guidance_rescale=0.0, _step=None, _rng_batch=None, **kwargs):
        self._check_step_options(use_original_steps, quantize_denoised, score_corrector)
        if cfg_img is None:
            cfg_img = unconditional_guidance_scale
        uc_img = kwargs['unconditional_conditioning_img_nonetext']           # KeyError like ddim_multiplecond.py:224
        step = int(t[0].item()) if _step is None else _step
        v_u = v_i = None
        if unconditional_conditioning is None or unconditional_guidance_scale == 1.:
            v_c = self.model.apply_model(x, t, c, **kwargs)
        else:
            if uc_img is None:
                raise ValueError("three-way CFG needs unconditional_conditioning_img_nonetext (image_guided_synthesis only builds it "
                                 "when cfg_img != 1.0, utils/diffusion_utils.py:157-163)")
            v_c, v_u, v_i = self._apply_three(x, t, c, unconditional_conditioning, uc_img, kwargs)
        sc = self.step_scalars(index, step)
        sc["cfg_scale"], sc["guidance_rescale"] = float(unconditional_guidance_scale), float(guidance_rescale)
        noise = self._step_noise(x, repeat_noise, temperature, noise_dropout, _rng_batch)
        return self._fused_update(x, v_c, v_u, noise, sc, v_uncond_img=v_i, cfg_img=float(cfg_img))

    def _apply_three(self, x, t, c, uc, uc_img, kwargs):
        """(v_cond, v_uncond, v_uncond_img) of one step (see the module docstring for the layouts)."""
        cfg = getattr(self.model, "_cfg", None)
        if cfg is not None:                                   # multi-GPU CFG split: branch 0 = cond, branch 1 = uncond | uncond_img
            if cfg.branch == 0:
                mine = self.model.apply_model(x, t, c, **kwargs)
            elif self._can_stack(uc, uc_img):
                mine = torch.cat(self._apply_stacked(x, t, (uc, uc_img), kwargs), 0)
            else:
                mine = torch.cat([self.model.apply_model(x, t, uc, **kwargs), self.model.apply_model(x, t, uc_img, **kwargs)], 0)
            b = x.shape[0]
            v_c, v_ui = cfg.exchange(mine.float().contiguous(), rows=(b, 2 * b))
            return v_c, v_ui[:b], v_ui[b:]
        if self._can_stack(c, uc, uc_img):
            return tuple(self._apply_stacked(x, t, (c, uc, uc_img), kwargs))
        v_c, v_u = self._apply_both(x, t, c, uc, kwargs)
        return v_c, v_u, self.model.apply_model(x, t, uc_img, **kwargs)
