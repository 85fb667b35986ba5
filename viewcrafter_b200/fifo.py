"""FIFO-Diffusion diagonal denoising (Kim et al., NeurIPS 2024) for clips of any length at the memory of one window
(INTEGRATION.md "Long clips: FIFO diagonal denoising").  New functionality: the reference samples a clip in one piece.

``FIFOSampler`` (two-way guidance, a ``ddim.DDIMSampler``) and ``FIFOSamplerMultiCond`` (three-way, a ``ddim_multiplecond.DDIMSampler``)
take DDIM's ``sample()`` arguments plus ``fifo_window=f`` and return ``(samples, intermediates)``.  ``shape[1]`` is the clip length N
and every ``c_concat`` entry carries all N frames.  With S DDIM steps and timesteps tau_0 < ... < tau_{S-1}, 2 <= f <= 128, S % f == 0:

  * N <= f: the ordinary sampler's call, bit for bit.
  * Warm start: frames [0, f) are sampled by the ordinary sampler of the same class with the same guidance (its draws at
    [B, 4, f, h, w]); call the result z.
  * Queue: eps = randn([B, 4, S, h, w]); position k holds sqrt(a(tau_k)) z[:, :, max(0, k - (S - f))] + sqrt(1 - a(tau_k)) eps[:, :, k].
  * At iteration m, position k holds render r = m + k - (S - f); its c_concat is the latent of render clamp(r, 0, N - 1).
  * Iteration m = 0 .. N + S - f - 1: for each partition p = 0 .. S/f - 1, the window of positions [p f, p f + f) gets one guided U-Net
    evaluation with per-frame timesteps tau_{p f .. p f + f - 1} (UNetModel.forward with [B, f] timesteps), a noise draw
    randn([B, 4, f, h, w]) (also at eta = 0, as DDIM draws it), and one ops.ddim_update_frames with index k's step_scalars at position
    k.  The head (position 0) is then clean: if its render m - (S - f) is >= 0 it is that output frame.  The queue shifts by one and
    randn([B, 4, 1, h, w]) enters at position S - 1, on every iteration including the last.  Partitions are disjoint, so each reads
    the latents from before the iteration.
  * Guidance rescale: per sample over the window [4, f, h, w] (DDIMSampler._fused_update's per-sample split), what the ordinary
    sampler computes for an f-frame clip.

The U-Net sees windows of f frames only, so memory does not depend on N; the steady-state cost is S / f forwards of f frames per output
frame, the per-frame cost of ordinary S-step sampling.  All partitions share one stacked cross-attention context tensor, so the U-Net's
K/V cache and its CUDA graph (keyed on that tensor's identity) serve every forward after the first two.
"""
from __future__ import annotations

import functools
import inspect

import torch

from . import ops
from . import ddim as _ddim
from . import ddim_multiplecond as _ddim_mc

# sample() options FIFO does not define: name -> test of the value that turns the option on
_UNSUPPORTED = {"mask": lambda v: v is not None, "x0": lambda v: v is not None, "x_T": lambda v: v is not None,
                "timesteps": lambda v: v is not None, "noise_dropout": lambda v: v > 0., "temperature": lambda v: v != 1.,
                "repeat_noise": bool, "score_corrector": lambda v: v is not None, "quantize_x0": bool,
                "_rng_rows": lambda v: v is not None}
MAX_WINDOW = 128            # the U-Net's temporal range
_COND_NAMES = ("conditioning", "unconditional_conditioning", "unconditional_conditioning_img_nonetext")


def check_window(f, steps: int) -> int:
    """f as an int; ValueError unless 2 <= f <= 128 and f divides the number of DDIM steps."""
    if isinstance(f, bool) or not isinstance(f, int) or not 2 <= f <= MAX_WINDOW:
        raise ValueError(f"FIFO window must be an int with 2 <= f <= {MAX_WINDOW}, got {f!r}")
    if steps % f:
        raise ValueError(f"FIFO needs the number of DDIM steps to be a multiple of the window: {steps} steps, window {f}")
    return f


class _FIFOMixin:
    """What FIFO adds to its DDIM base class (first in the MRO).  The class's own p_sample_ddim runs each window's guided forwards and
    noise draw; _fused_update swaps the update for ops.ddim_update_frames with the window's per-frame scalars, and _stacked_conditioning
    keeps one stacked context tensor while the windows' c_concat changes."""
    _fifo_frames = None         # per-frame step scalars of the window being updated (while sample() runs the queue)
    _fifo_ctx = None            # stacked context tensors by the ids of the branches' c_crossattn entries (while sample() runs the queue)

    @torch.no_grad()
    def sample(self, *args, fifo_window=None, **kwargs):
        """DDIMSampler.sample's arguments plus fifo_window=f (module docstring).  shape = (C, N, h, w).  Raises ValueError for a bad
        window or shape and NotImplementedError for mask, x0, x_T, timesteps, noise_dropout > 0, temperature != 1, repeat_noise,
        score_corrector and quantize_x0, before any forward.  Returns (samples [B, C, N, h, w], {"x_inter": [samples],
        "pred_x0": [samples]}); callback(m) is called after every queue iteration (not in the warm start), img_callback is not called."""
        bound = inspect.signature(_ddim.DDIMSampler.sample).bind(self, *args, **kwargs).arguments
        given = dict(bound, **bound.get("kwargs", {}))
        for name, on in _UNSUPPORTED.items():
            if name in given and on(given[name]):
                raise NotImplementedError(f"{type(self).__name__}: sample({name}=...) is not supported by FIFO diagonal denoising")
        shape = tuple(given["shape"])
        if len(shape) != 4:
            raise ValueError(f"{type(self).__name__}: FIFO samples a clip, shape must be (C, N, h, w), got {shape}")
        spacing = given.get("timestep_spacing", "uniform")
        self.make_schedule(ddim_num_steps=given["S"], ddim_discretize=spacing, ddim_eta=given.get("eta", 0.), verbose=False)
        S = len(self.ddim_timesteps)
        f = check_window(fifo_window, S)
        N = shape[1]
        if N <= f:
            return super().sample(*args, **kwargs)
        for name in _COND_NAMES:
            cond = given.get(name)
            for src in (cond.get("c_concat", []) if isinstance(cond, dict) else []):
                if src.dim() != 5 or src.shape[2] != N:
                    raise ValueError(f"{type(self).__name__}: every c_concat entry must carry all {N} frames, got {tuple(src.shape)}")
        slice_frames = _frame_slicer()
        warm = {k: v for k, v in given.items() if k not in ("self", "kwargs", "callback", "img_callback")}
        warm.update(shape=(shape[0], f, *shape[2:]), conditioning=slice_frames(given.get("conditioning"), 0, f),
                    unconditional_conditioning=slice_frames(given.get("unconditional_conditioning"), 0, f))
        if "unconditional_conditioning_img_nonetext" in warm:
            warm["unconditional_conditioning_img_nonetext"] = slice_frames(warm["unconditional_conditioning_img_nonetext"], 0, f)
        z, _ = super().sample(**warm)
        try:
            samples = self._run_queue(z, given, S, f, N)
        finally:
            self._fifo_frames = self._fifo_ctx = None
        return samples, {"x_inter": [samples], "pred_x0": [samples]}

    def _run_queue(self, z, given, S, f, N):
        B, C, _, h, w = z.shape
        dev = z.device
        steps = [int(t) for t in self.ddim_timesteps]
        eps = torch.randn((B, C, S, h, w), device=dev)
        queue = torch.empty((B, C, S, h, w), device=dev, dtype=torch.float32)
        for k in range(S):
            zk = z[:, :, max(0, k - (S - f))].float()
            queue[:, :, k] = float(self._sqrt_ac[steps[k]]) * zk + float(self._sqrt_1mac[steps[k]]) * eps[:, :, k]
        del eps
        out = torch.empty((B, C, N, h, w), device=dev, dtype=torch.float32)
        # per partition: its [B, f] timesteps, its per-frame step scalars and the guidance branches with c_concat buffers of f frames
        # that are refilled every iteration
        parts = []
        gather = _ConcatGather(f)
        for p in range(S // f):
            ks = range(p * f, p * f + f)
            t = torch.tensor([steps[k] for k in ks], device=dev, dtype=torch.long).repeat(B, 1)
            frames = [self.step_scalars(k, steps[k]) for k in ks]
            conds = {n: gather.branch(given.get(n), p) for n in _COND_NAMES}
            parts.append((t, frames, conds))
        extra = {k: v for k, v in given.get("kwargs", {}).items() if k not in ("window_seed", "clean_cond")}
        base = (torch.arange(S, device=dev) - (S - f))
        self._fifo_ctx = {}
        callback = given.get("callback")
        for m in range(N + S - f):
            for p, (t, frames, conds) in enumerate(parts):
                sl = slice(p * f, p * f + f)
                gather.fill(p, (base[sl] + m).clamp_(0, N - 1))
                kw = dict(extra, unconditional_guidance_scale=given.get("unconditional_guidance_scale", 1.),
                          unconditional_conditioning=conds["unconditional_conditioning"], fs=given.get("fs"),
                          guidance_rescale=given.get("guidance_rescale", 0.0), corrector_kwargs=given.get("corrector_kwargs"))
                if "unconditional_conditioning_img_nonetext" in extra:
                    kw["unconditional_conditioning_img_nonetext"] = conds["unconditional_conditioning_img_nonetext"]
                self._fifo_frames = frames
                queue[:, :, sl], _ = self.p_sample_ddim(queue[:, :, sl].contiguous(), conds["conditioning"], t, index=p * f,
                                                        _step=steps[p * f], **kw)
            if m >= S - f:
                out[:, :, m - (S - f)] = queue[:, :, 0]
            queue = torch.cat([queue[:, :, 1:], torch.randn((B, C, 1, h, w), device=dev)], 2)
            if callback:
                callback(m)
        return out

    def _fused_update(self, x, v_c, v_u, noise, sc, **extra):
        """DDIM's fused update; inside the queue, ops.ddim_update_frames with the window's per-frame scalars (sc keeps the per-call
        cfg_scale and guidance_rescale), split per sample under guidance rescale like the ordinary update."""
        if self._fifo_frames is None:
            return super()._fused_update(x, v_c, v_u, noise, sc, **extra)
        op = functools.partial(ops.ddim_update_frames, frames=self._fifo_frames)
        return _ddim.DDIMSampler._fused_update(x, v_c, v_u, noise, sc, op=op, **extra)

    def _stacked_conditioning(self, *conds):
        """Inside the queue: the stacked c_crossattn is built once per tuple of branch contexts and kept as the same tensors for every
        window and iteration (the U-Net keys its K/V cache and graphs on the context object); c_concat, refilled in place every
        iteration, is stacked anew on every call."""
        if self._fifo_ctx is None:
            return super()._stacked_conditioning(*conds)
        cat = {}
        for k in conds[0]:
            groups = list(zip(*(c[k] for c in conds)))
            if k == "c_concat":
                cat[k] = [torch.cat(list(ents), 0) for ents in groups]
                continue
            key = (k,) + tuple(id(a) for ents in groups for a in ents)
            if key not in self._fifo_ctx:
                self._fifo_ctx[key] = (groups, [torch.cat(list(ents), 0) for ents in groups])     # keeps the sources alive
            cat[k] = self._fifo_ctx[key][1]
        same = "c_concat" in conds[0] and all(a is u for ents in zip(*(c["c_concat"] for c in conds)) for a, u in zip(ents, ents[1:]))
        return cat, same

    def decode(self, *args, **kwargs):
        raise NotImplementedError(f"{type(self).__name__}.decode: the img2img helper is DDIM's; use ddim.DDIMSampler")


def _frame_slicer():
    """slice(cond, lo, hi): the conditioning dict with every c_concat entry cut to frames [lo, hi).  Entries that share a tensor share
    its slice, so the branches keep the shared c_concat the CFG prefix sharing relies on."""
    memo = {}

    def cut(t, lo, hi):
        key = (id(t), lo, hi)
        if key not in memo:
            memo[key] = t[:, :, lo:hi]
        return memo[key]

    def slice_frames(cond, lo, hi):
        if not isinstance(cond, dict) or "c_concat" not in cond:
            return cond
        return dict(cond, c_concat=[cut(t, lo, hi) for t in cond["c_concat"]])
    return slice_frames


class _ConcatGather:
    """Per partition, one f-frame buffer per distinct c_concat source tensor (branches that share a source share its buffer), refilled
    in place with the renders of the window's positions."""

    def __init__(self, f):
        self.f = f
        self.bufs = {}              # (partition, id(source)) -> (source, buffer)

    def branch(self, cond, p):
        if not isinstance(cond, dict) or "c_concat" not in cond:
            return cond
        ents = []
        for src in cond["c_concat"]:
            key = (p, id(src))
            if key not in self.bufs:
                self.bufs[key] = (src, torch.empty((src.shape[0], src.shape[1], self.f, *src.shape[3:]), device=src.device, dtype=src.dtype))
            ents.append(self.bufs[key][1])
        return dict(cond, c_concat=ents)

    def fill(self, p, idx):
        for (q, _), (src, buf) in self.bufs.items():
            if q == p:
                torch.index_select(src, 2, idx.to(src.device), out=buf)


class FIFOSampler(_FIFOMixin, _ddim.DDIMSampler):
    """FIFO diagonal denoising with two-way guidance (image_guided_synthesis(..., fifo=f))."""


class FIFOSamplerMultiCond(_FIFOMixin, _ddim_mc.DDIMSampler):
    """FIFO diagonal denoising with three-way guidance (image_guided_synthesis(..., fifo=f, multiple_cond_cfg=True))."""
