"""Caller of the hot path: ``get_latent_z`` / ``image_guided_synthesis`` (reference: utils/diffusion_utils.py:110-201) --
SURVEY.md 8(f) rank f2.

Same signature, conditioning construction, RNG order and return layout (``[batch, n_samples, c, t, h, w]``) as the
reference function, which ``viewcrafter.py:run_diffusion`` (viewcrafter.py:92-107) calls once per clip.  ``model`` is the
reference's ``VIPLatentDiffusion`` (with the U-Net / VAE / image_proj_model swapped for the viewcrafter_b200 classes by the
YAML ``target:`` lines, INTEGRATION.md) or any object with the same attributes: ``embedder``, ``image_proj_model``,
``get_learned_conditioning``, ``encode_first_stage``, ``decode_first_stage``, ``uncond_type``, ``model.conditioning_key``.

What differs from the reference, all parity-preserving (SURVEY.md App. C):
  * the sampler is created with ``batch_cfg=True``: cond + uncond run as one B=2 U-Net forward with the context-free prefix
    computed once, and -- because the same ``cond`` / ``uc`` tensors are handed to every step and every ``n_samples``
    iteration -- the cross-attention K/V projections are computed once per clip;
  * ``cuda_graph=True`` lets the viewcrafter_b200 U-Net replay its forward as one captured CUDA graph from the third call on
    (``UNetModel.enable_cuda_graph``): same kernels in the same order, ~1000 launches -> 1 per forward;
  * on a model sharded by ``parallel.shard_model`` the VAE encode and decode run frame-sharded over all ranks (same latents, same
    posterior draws in the same order, same decoded frames; INTEGRATION.md "Multi-GPU");
  * on a model sharded with ``shard_model(replicas=R > 1)`` the ``n_samples`` x batch outputs run concurrently on R GPU groups, each
    with the random numbers the single process draws for it, and are decoded together over all ranks (``_sample_on_replicas``);
  * nothing else: conditioning tensors, ``x_T`` / per-step noise draws and the decode are the reference's, in its order.
"""
from __future__ import annotations

import contextlib

import torch

from . import fifo as _fifo
from . import ops, parallel, temporal_window as _tw
from .ddim import DDIMSampler, check_row_replay
from .ddim_multiplecond import DDIMSampler as DDIMSampler_multicond
from .dpm_solver import DPMSolver3MSDESampler, DPMSolver3MSDESamplerMultiCond, DPMSolverSampler, DPMSolverSamplerMultiCond

# image_guided_synthesis(sampler=...) -> (two-way sampler class, three-way sampler class)
SAMPLERS = {"ddim": (DDIMSampler, DDIMSampler_multicond), "dpmpp_2m": (DPMSolverSampler, DPMSolverSamplerMultiCond),
            "dpmpp_3m_sde": (DPMSolver3MSDESampler, DPMSolver3MSDESamplerMultiCond)}


def _vae_sharded(model) -> bool:
    """True when parallel.shard_model gave the model a VAE communicator over more than one rank."""
    return bool(getattr(model, "_vae_comm", None))


def get_latent_z(model, videos):
    """videos [b, c, t, h, w] -> latents [b, c', t, h/8, w/8] via per-frame encode_first_stage (diffusion_utils.py:110-115).
    On a model sharded by parallel.shard_model the frames are encoded over all ranks (parallel.vae_encode), same latents."""
    if _vae_sharded(model):
        return parallel.vae_encode(model, videos)
    b, c, t, h, w = videos.shape
    x = videos.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
    z = model.encode_first_stage(x)
    return z.reshape(b, t, *z.shape[1:]).permute(0, 2, 1, 3, 4)


@torch.no_grad()
def image_guided_synthesis(model, prompts, videos, noise_shape, n_samples=1, ddim_steps=50, ddim_eta=1.,
                           unconditional_guidance_scale=1.0, cfg_img=None, fs=None, text_input=False, multiple_cond_cfg=False,
                           timestep_spacing='uniform', guidance_rescale=0.0, condition_index=None, batch_cfg=True, cuda_graph=True,
                           reproducible=None, sampler="ddim", temporal_window=None, window_seed=0, fifo=None, **kwargs):
    """reproducible: True / False switches viewcrafter_b200's reproducible mode (ops.set_reproducible) for this call and restores the
    previous setting afterwards; None leaves the process setting as it is.
    sampler: "ddim" (the reference's DDIMSampler), "dpmpp_2m" (dpm_solver.DPMSolverSampler / DPMSolverSamplerMultiCond, which takes
    ddim_eta 0 or 1 only) or "dpmpp_3m_sde" (dpm_solver.DPMSolver3MSDESampler / DPMSolver3MSDESamplerMultiCond, ddim_eta 1 only;
    INTEGRATION.md "Samplers").
    temporal_window: None (full temporal attention) or (W, S): the U-Net runs windowed temporal attention for this call and the drawn
    x_T is rescheduled with window_seed (FreeNoise; INTEGRATION.md "Long clips: windowed temporal attention").  The U-Net's previous
    setting is restored afterwards.  An explicit x_T= is used as given, without rescheduling.
    fifo: None, or a window f (2 <= f <= 128, ddim_steps a multiple of f): FIFO-Diffusion's diagonal denoising (fifo.FIFOSampler /
    FIFOSamplerMultiCond; INTEGRATION.md "Long clips: FIFO diagonal denoising").  videos and noise_shape carry all N frames while the
    U-Net only ever runs on f of them, so memory does not grow with N; the latents are decoded f frames at a time.  It runs with
    sampler="ddim" only, without temporal_window and not on replica groups (ValueError before any work)."""
    if sampler not in SAMPLERS:
        raise ValueError(f"unknown sampler {sampler!r}; choose one of {sorted(SAMPLERS)}")
    if fifo is not None:
        if sampler != "ddim":
            raise ValueError(f"image_guided_synthesis: fifo runs with sampler='ddim' only, got sampler={sampler!r}")
        if temporal_window is not None:
            raise ValueError("image_guided_synthesis: fifo and temporal_window cannot be combined (FIFO's U-Net windows are full clips)")
        if getattr(model, "_replicas", None) is not None:
            raise ValueError("image_guided_synthesis: fifo does not run on replica groups (parallel.shard_model(replicas=R > 1))")
        _fifo.check_window(fifo, ddim_steps)
        kwargs["fifo_window"] = fifo
    if sampler != "ddim":
        SAMPLERS[sampler][0].check_eta(ddim_eta)          # before the conditioning is computed
    with _unet_window(model, _tw.check_window(temporal_window)):
        if reproducible is None:
            return _synthesis(model, prompts, videos, noise_shape, n_samples, ddim_steps, ddim_eta, unconditional_guidance_scale, cfg_img,
                              fs, text_input, multiple_cond_cfg, timestep_spacing, guidance_rescale, condition_index, batch_cfg, cuda_graph,
                              sampler=sampler, window_seed=window_seed, **kwargs)
        prev = ops.set_reproducible(reproducible)
        try:
            return _synthesis(model, prompts, videos, noise_shape, n_samples, ddim_steps, ddim_eta, unconditional_guidance_scale, cfg_img,
                              fs, text_input, multiple_cond_cfg, timestep_spacing, guidance_rescale, condition_index, batch_cfg, cuda_graph,
                              sampler=sampler, window_seed=window_seed, **kwargs)
        finally:
            ops.set_reproducible(prev)


@contextlib.contextmanager
def _unet_window(model, window):
    """The U-Net's temporal window set to `window` (None: off) inside the block and restored after it."""
    unet = getattr(getattr(model, "model", None), "diffusion_model", None)
    if not hasattr(unet, "set_temporal_window"):
        if window is not None:
            raise ValueError("image_guided_synthesis: temporal_window needs the viewcrafter_b200 UNetModel")
        yield
        return
    prev = unet.temporal_window
    unet.set_temporal_window(window)
    try:
        yield
    finally:
        unet.set_temporal_window(prev)


def _synthesis(model, prompts, videos, noise_shape, n_samples, ddim_steps, ddim_eta, unconditional_guidance_scale, cfg_img, fs, text_input,
               multiple_cond_cfg, timestep_spacing, guidance_rescale, condition_index, batch_cfg, cuda_graph, sampler="ddim", **kwargs):
    if getattr(model, "_replicas", None) is not None:
        check_row_replay(kwargs)                          # before any collective, on every rank alike
    unet = getattr(getattr(model, "model", None), "diffusion_model", None)
    if cuda_graph and hasattr(unet, "enable_cuda_graph") and next(unet.parameters()).is_cuda:
        unet.enable_cuda_graph()              # the ~100 forwards of a clip share shapes, weights and context: capture once, replay
    fifo = kwargs.get("fifo_window")
    classes = (_fifo.FIFOSampler, _fifo.FIFOSamplerMultiCond) if fifo is not None else SAMPLERS[sampler]
    ddim_sampler = classes[bool(multiple_cond_cfg)](model, batch_cfg=batch_cfg)
    batch_size = noise_shape[0]
    fs = torch.tensor([fs] * batch_size, dtype=torch.long, device=model.device)

    if not text_input:
        prompts = [""] * batch_size
    assert condition_index is not None, "Error: condition index is None!"

    img = videos[:, :, condition_index[0]]                                   # b c h w
    img_emb = model.image_proj_model(model.embedder(img))                   # b l c
    cond_emb = model.get_learned_conditioning(prompts)
    cond = {"c_crossattn": [torch.cat([cond_emb, img_emb], dim=1)]}
    hybrid = model.model.conditioning_key == 'hybrid'
    if hybrid:
        img_cat_cond = get_latent_z(model, videos)                           # b c t h w
        cond["c_concat"] = [img_cat_cond]

    uc = None
    if unconditional_guidance_scale != 1.0:
        if model.uncond_type == "empty_seq":
            uc_emb = model.get_learned_conditioning(batch_size * [""])
        elif model.uncond_type == "zero_embed":
            uc_emb = torch.zeros_like(cond_emb)
        else:
            raise ValueError(f"unknown uncond_type {model.uncond_type!r}")
        uc_img_emb = model.image_proj_model(model.embedder(torch.zeros_like(img)))
        uc = {"c_crossattn": [torch.cat([uc_emb, uc_img_emb], dim=1)]}
        if hybrid:
            uc["c_concat"] = [img_cat_cond]                                  # the SAME tensor as cond's: enables the shared CFG prefix

    # one more unconditional branch for the three-way CFG: image kept, text dropped (diffusion_utils.py:157-165)
    if multiple_cond_cfg and cfg_img != 1.0:
        uc_2 = {"c_crossattn": [torch.cat([uc_emb, img_emb], dim=1)]}
        if hybrid:
            uc_2["c_concat"] = [img_cat_cond]
        kwargs.update({"unconditional_conditioning_img_nonetext": uc_2})
    else:
        kwargs.update({"unconditional_conditioning_img_nonetext": None})

    options = dict(S=ddim_steps, batch_size=batch_size, shape=noise_shape[1:], verbose=False,
                   unconditional_guidance_scale=unconditional_guidance_scale, eta=ddim_eta, cfg_img=cfg_img, mask=None, x0=None,
                   timestep_spacing=timestep_spacing, guidance_rescale=guidance_rescale, **kwargs)
    replicas = getattr(model, "_replicas", None)
    if replicas is not None:
        return _sample_on_replicas(model, replicas, ddim_sampler, cond, uc, fs, n_samples, options)
    batch_variants = []
    for _ in range(n_samples):
        samples, _ = ddim_sampler.sample(conditioning=cond, unconditional_conditioning=uc, fs=fs, **options)
        # latent -> pixel space; on a sharded model every rank decodes its share of the frames (parallel.vae_decode).  FIFO clips are
        # decoded at most f frames at a time, so the decoder's activations do not grow with the clip either
        decode = (lambda z: parallel.vae_decode(model, z)) if _vae_sharded(model) else model.decode_first_stage
        if fifo is None:
            batch_variants.append(decode(samples))
        else:
            batch_variants.append(torch.cat([decode(samples[:, :, i:i + fifo]) for i in range(0, samples.shape[2], fifo)], 2))
    return torch.stack(batch_variants).permute(1, 0, 2, 3, 4, 5)              # batch, variants, c, t, h, w


def _rows(conds, b):
    """Row b of the conditioning dicts `conds` (None stays None).  Every tensor is sliced once, so entries that share a tensor (the
    c_concat of all branches) share its slice: the shared CFG prefix, the U-Net's K/V cache and its graph key rely on that identity."""
    memo = {}

    def row(t):
        if id(t) not in memo:
            memo[id(t)] = t[b:b + 1]
        return memo[id(t)]
    return [None if c is None else {k: [row(t) for t in v] for k, v in c.items()} for c in conds]


def _sample_on_replicas(model, replicas, sampler, cond, uc, fs, n_samples, options):
    """The sampling and decode of image_guided_synthesis on a model sharded with shard_model(replicas=R > 1).  The n_samples x B
    outputs are independent jobs j = k * B + b (sample k, clip b); group j % R runs job j as rows (b, b + 1) of sample k's batch
    (DDIMSampler.sample(_rng_rows=...)), with the random numbers a single process draws for that batch.  The job latents are gathered
    over the world and all n_samples * B clips are decoded in one parallel.vae_decode over all ranks.  Returns [B, n_samples, c, t, h, w]
    on every rank, and leaves the device generator in the state a single process leaves it in."""
    B = options["batch_size"]
    n_jobs = n_samples * B
    mine = replicas.jobs(n_jobs)
    device = sampler._device()
    if device.type == "cuda":
        get_state, set_state = (lambda: torch.cuda.get_rng_state(device)), (lambda s: torch.cuda.set_rng_state(s, device))
    else:
        get_state, set_state = torch.get_rng_state, torch.set_rng_state
    # a single process draws x_T and every step's noise of sample 0, then of sample 1, ...: walk that stream once, keeping the
    # generator state at the start of every sample this group has a job in
    starts = {}
    for k in range(n_samples):
        if any(j // B == k for j in mine):
            starts[k] = get_state()
        sampler.skip_sample_draws(options["S"], (B, *options["shape"]), device, options["timestep_spacing"])
    end = get_state()
    clips, latents = {}, []
    for j in mine:
        k, b = divmod(j, B)
        if b not in clips:                 # one sampler per clip: its stacked conditioning (and the U-Net graph) is reused by every job
            c, u, u2 = _rows((cond, uc, options["unconditional_conditioning_img_nonetext"]), b)
            clips[b] = (type(sampler)(model, batch_cfg=sampler.batch_cfg),
                        dict(options, conditioning=c, unconditional_conditioning=u, unconditional_conditioning_img_nonetext=u2, fs=fs[b:b + 1]))
        smp, kw = clips[b]
        set_state(starts[k])
        z, _ = smp.sample(_rng_rows=(b, b + 1), **kw)
        latents.append(z)
    set_state(end)
    z = replicas.gather_jobs(latents, n_jobs, tuple(options["shape"]), device)
    y = parallel.vae_decode(model, z) if _vae_sharded(model) else model.decode_first_stage(z)
    return y.reshape(n_samples, B, *y.shape[1:]).permute(1, 0, 2, 3, 4, 5)
