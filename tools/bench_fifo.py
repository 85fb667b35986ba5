#!/usr/bin/env python
"""FIFO-Diffusion diagonal denoising at 576x1024 on one GPU: time per output frame, time per clip and peak memory against the clip length,
next to ordinary DDIM.

    python tools/bench_fifo.py [--frames 49,128,256,512] [--window 25] [--steps 50] [--ddim-frames 49,128] [--ddim-steps 10]

bench.py's random-weight full-width model with a random-weight VAE decoder, two-way guidance with batch_cfg and graph replay (CFG 7.5,
rescale 0.7, eta 1, uniform_trailing, fs 10), random render latents and contexts.
1. For every N of --frames: fifo.FIFOSampler.sample(fifo_window=--window, S=--steps) then the decode in chunks of `window` frames.
   Reports the steady-state seconds per output frame (the mean queue iteration after the first three, each iteration ending in a
   device synchronise; one iteration outputs one frame), the seconds per clip (warm start + queue + decode, host clock around work that
   ends in a synchronise; the VAE encode and the conditioning are not included) and torch.cuda.max_memory_allocated.
2. For every N of --ddim-frames: ordinary ddim.DDIMSampler steps on the whole clip (2 untimed steps, then --ddim-steps timed with CUDA
   events), reported as seconds per step, the per-output-frame cost of a 50-step clip (50 s/step / N) and the peak memory.
A configuration that runs out of device memory is recorded as such and the others still run.  Prints one JSON line per configuration and
a last line with all of them, the card name and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H, W = 72, 128                 # 576x1024 latents


def _inputs(N, device):
    g = torch.Generator().manual_seed(2)
    cc = torch.randn(1, 4, N, H, W, generator=g).to(device)
    c, uc = ({"c_crossattn": [torch.randn(1, 333, 1024, generator=g).to(device)], "c_concat": [cc]} for _ in range(2))
    return c, uc


def _oom(e):
    return ". ".join(str(e).split(". ")[:2]) + "."                 # "CUDA out of memory. Tried to allocate ..."


def fifo_run(model, N, window, steps):
    from viewcrafter_b200 import fifo
    device = torch.device("cuda")
    c, uc = _inputs(N, device)
    fs = torch.tensor([10], device=device)
    ticks = []

    def tick(m):
        torch.cuda.synchronize()
        ticks.append(time.perf_counter())
        if m % 50 == 49:
            print(f"N={N}: iteration {m + 1} of {N + steps - window}", file=sys.stderr, flush=True)

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(0)
    t0 = time.perf_counter()
    z, _ = fifo.FIFOSampler(model, batch_cfg=True).sample(
        S=steps, batch_size=1, shape=(4, N, H, W), conditioning=c, unconditional_conditioning=uc, unconditional_guidance_scale=7.5,
        eta=1.0, guidance_rescale=0.7, timestep_spacing="uniform_trailing", fs=fs, verbose=False, fifo_window=window, callback=tick)
    torch.cuda.synchronize()
    t_sample = time.perf_counter() - t0
    video = torch.cat([model.decode_first_stage(z[:, :, i:i + window]) for i in range(0, N, window)], 2)
    torch.cuda.synchronize()
    t_clip = time.perf_counter() - t0
    its = np.diff(ticks)[3:] if len(ticks) > 4 else np.diff(ticks)
    return dict(sampler="fifo", N=N, window=window, steps=steps, iterations=len(ticks),
                s_per_output_frame=round(float(its.mean()), 4) if len(its) else None,
                s_sampling=round(t_sample, 2), s_per_clip=round(t_clip, 2), peak_GB=round(torch.cuda.max_memory_allocated() / 1e9, 2),
                finite=bool(torch.isfinite(video).all()), video_shape=list(video.shape))


def ddim_run(model, N, steps_timed):
    from viewcrafter_b200 import ddim
    device = torch.device("cuda")
    c, uc = _inputs(N, device)
    fs = torch.tensor([10], device=device)
    sampler = ddim.DDIMSampler(model, batch_cfg=True)
    sampler.make_schedule(50, "uniform_trailing", 1.0, verbose=False)
    order = np.flip(sampler.ddim_timesteps)
    x = torch.randn(1, 4, N, H, W, device=device)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()

    def step(x, i):
        ts = torch.full((1,), int(order[i]), device=device, dtype=torch.long)
        return sampler.p_sample_ddim(x, c, ts, index=50 - i - 1, unconditional_guidance_scale=7.5, unconditional_conditioning=uc,
                                     fs=fs, guidance_rescale=0.7, _step=int(order[i]))[0]

    for i in range(2):
        x = step(x, i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps_timed):
        x = step(x, 2 + i)
    e1.record()
    torch.cuda.synchronize()
    s_step = e0.elapsed_time(e1) * 1e-3 / steps_timed
    return dict(sampler="ddim", N=N, s_per_step=round(s_step, 4), s_per_output_frame_50_steps=round(50 * s_step / N, 4),
                peak_GB=round(torch.cuda.max_memory_allocated() / 1e9, 2), finite=bool(torch.isfinite(x).all()))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", default="49,128,256,512")
    ap.add_argument("--window", type=int, default=25)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--ddim-frames", default="49,128")
    ap.add_argument("--ddim-steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fifo.py measures on a CUDA device; none is available")
    import bench
    from bench_multicond import card
    from viewcrafter_b200.autoencoder import AutoencoderKL
    from viewcrafter_b200.configs import VAE_DDCONFIG
    torch.cuda.set_device(0)
    model = bench.build_model(bench.WORKLOADS["ViewCrafter_25"], torch.device("cuda"))
    model.first_stage_model = AutoencoderKL(VAE_DDCONFIG, None, 4).eval()
    model = model.cuda()                          # the schedule buffers too: the samplers draw on the device of model.betas
    unet = model.model.diffusion_model
    unet.enable_cuda_graph()
    runs = []
    configs = [("fifo", int(n)) for n in args.frames.split(",") if n] + [("ddim", int(n)) for n in args.ddim_frames.split(",") if n]
    for kind, N in configs:
        try:
            with torch.no_grad():
                r = fifo_run(model, N, args.window, args.steps) if kind == "fifo" else ddim_run(model, N, args.ddim_steps)
        except torch.OutOfMemoryError as e:
            r = dict(sampler=kind, N=N, out_of_memory=_oom(e))
        unet.enable_cuda_graph(False).enable_cuda_graph()          # drop this configuration's graphs
        torch.cuda.empty_cache()
        if "out_of_memory" in r:
            r["peak_GB"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
        runs.append(r)
        print(json.dumps(r), flush=True)
    name, power = card()
    print(json.dumps({"metric": f"FIFO diagonal denoising at 576x1024 (1 GPU, two-way batch_cfg, graph replay, window {args.window}, "
                                f"{args.steps} steps)", "runs": runs, "card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
