#!/usr/bin/env python
"""Clip length on one GPU at 576x1024: DDIM steps/s and peak memory per frame count, the longest clip that fits, and the
temporal-attention kernel alone.

    python tools/bench_long_clip.py [--frames 25,49,64,96] [--steps 5] [--warmup 2] [--reps 200]

1. For every T of --frames, two-way (B = 2) and three-way (B = 3) guidance: steps/s of ddim.DDIMSampler / ddim_multiplecond.DDIMSampler
   with batch_cfg and graph replay (CFG 7.5, cfg_img 2.0, rescale 0.7, eta 1) on bench.py's random-weight full-width model, timed
   with CUDA events over --steps steps after --warmup, and the peak torch.cuda.max_memory_allocated of that configuration.
2. Peak memory grows linearly in T (activations are rows of T * H * W); before a configuration runs, its peak is predicted (from one
   measured point: in proportion to T; from two or more: a least-squares line).  The line through the measured peaks of each B
   predicts the largest T whose peak stays under 90 % of what this process can allocate (free memory at the start plus what
   it held then).  A configuration of the list predicted not to fit is skipped and reported as such: the GPU is shared, so the limit
   is never found by running out of memory.  That T, capped at the kernel's 128 frames, runs once (warm-up + one timed step) to
   confirm it.
3. temporal_attn alone at level 0 (72 x 128 sites, 5 heads) and level 1 (36 x 64 sites, 10 heads), B = 2, for T = 25 (the T <= 32
   kernel) and T = 49 (the long-clip kernel) in the same run: device time per call over --reps launches (CUDA events) and the rate of
   its algorithmic bytes, 4 * B * T * sites * heads * 64 * 2 (q, k, v read once, out written once).
Prints one JSON line with every number, the card name and its power limit.

    python tools/bench_long_clip.py --window W,S [--frames 49,128] [--steps 3] [--warmup 2] [--reps 50]

runs the windowed temporal attention (UNetModel.set_temporal_window) instead: two-way steps/s and peak memory for every T of --frames
with the window and, where full attention exists (T <= 128), without it.  A configuration that runs out of device memory is recorded
as such (with the allocator's message) and the remaining ones still run; then the kernel alone at level 0 (B = 2) for T = 49 and 128,
windowed against the full kernels, with the algorithmic bytes 4 * T * 128 per (site, head) pair (each q, k, v row read once, each
output row written once).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H, W = 72, 128                 # 576x1024 latents
MAX_T = 128


def time_steps(model, B, T, steps, warmup):
    """(steps/s, peak bytes, finite) of `steps` guided DDIM steps at B = 2 (two-way) or 3 (three-way) guidance branches."""
    from viewcrafter_b200 import ddim, ddim_multiplecond
    device = torch.device("cuda")
    unet = model.model.diffusion_model
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 4, T, H, W, generator=g).to(device)
    cc = torch.randn(1, 4, T, H, W, generator=g).to(device)
    c, uc, ui = ({"c_crossattn": [torch.randn(1, 333, 1024, generator=g).to(device)], "c_concat": [cc]} for _ in range(3))
    sampler = (ddim_multiplecond if B == 3 else ddim).DDIMSampler(model, batch_cfg=True)
    sampler.make_schedule(50, "uniform_trailing", 1.0, verbose=False)
    kw = dict(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui) if B == 3 else {}
    fs = torch.tensor([10], device=device)
    order = np.flip(sampler.ddim_timesteps)
    unet.enable_cuda_graph()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()

    def step(x, i):
        i = i % 50
        ts = torch.full((1,), int(order[i]), device=device, dtype=torch.long)
        return sampler.p_sample_ddim(x, c, ts, index=50 - i - 1, unconditional_guidance_scale=7.5, unconditional_conditioning=uc,
                                     fs=fs, guidance_rescale=0.7, _step=int(order[i]), **kw)[0]

    torch.manual_seed(0)
    for i in range(warmup):
        x = step(x, i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        x = step(x, warmup + i)
    e1.record()
    torch.cuda.synchronize()
    rate = steps / (e0.elapsed_time(e1) * 1e-3)
    peak = torch.cuda.max_memory_allocated()
    finite = bool(torch.isfinite(x).all())
    unet.enable_cuda_graph(False)                       # drops the captured graphs and their memory pools
    del x, cc, c, uc, ui, sampler
    torch.cuda.empty_cache()
    return rate, peak, finite


def kernel_rate(B, T, sites, heads, reps, window=None):
    from viewcrafter_b200 import ops
    C = heads * 64
    g = torch.Generator(device="cuda").manual_seed(T)
    qkv = torch.randn(B * T * sites, 3 * C, generator=g, device="cuda").half()
    a = torch.empty(B * T * sites, C, device="cuda", dtype=torch.float16)

    def call():
        for b in range(B):                             # the U-Net's call sequence: one launch per batch element
            rows = slice(b * T * sites, (b + 1) * T * sites)
            if window is None:
                ops.temporal_attn(qkv[rows, :C], qkv[rows, C:2 * C], qkv[rows, 2 * C:], T, sites, heads, out=a[rows])
            else:
                ops.temporal_attn_windowed(qkv[rows, :C], qkv[rows, C:2 * C], qkv[rows, 2 * C:], T, sites, heads, *window, out=a[rows])

    for _ in range(5):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    dt = e0.elapsed_time(e1) * 1e-3 / reps
    nbytes = 4 * B * T * sites * heads * 64 * 2
    kernel = f"windowed{tuple(window)}" if window is not None else "T<=32" if T <= 32 else "33..128"
    return dict(level_sites=sites, heads=heads, B=B, T=T, kernel=kernel, us=round(dt * 1e6, 2), GB_per_s=round(nbytes / dt / 1e9, 1),
                bytes=nbytes)


def window_main(args, window):
    import bench
    from bench_multicond import card
    torch.cuda.set_device(0)
    frames = sorted(int(t) for t in (args.frames or "49,128").split(","))
    res = {"metric": f"windowed temporal attention {window} at 576x1024 (1 GPU, two-way batch_cfg, graph replay)", "kernel": []}
    for T in (49, 128):
        for w in (None, window):
            res["kernel"].append(kernel_rate(2, T, H * W, 5, args.reps, w))
            print(json.dumps(res["kernel"][-1]), flush=True)
    torch.cuda.empty_cache()
    model = bench.build_model(bench.WORKLOADS["ViewCrafter_25"], torch.device("cuda"))
    unet = model.model.diffusion_model
    runs = []
    for T in frames:
        for w in ((None, window) if T <= MAX_T else (window,)):
            unet.set_temporal_window(w)
            oom = None
            try:
                rate, peak, finite = time_steps(model, 2, T, args.steps, args.warmup)
            except torch.OutOfMemoryError as e:
                oom = ". ".join(str(e).split(". ")[:2]) + "."       # "CUDA out of memory. Tried to allocate ..."
            if oom is None:
                runs.append(dict(B=2, T=T, window=w, steps_per_s=round(rate, 4), peak_GB=round(peak / 1e9, 2), finite=finite))
            else:                                          # the exception and its frames are gone: release the graphs and the cache
                unet.enable_cuda_graph(False)
                torch.cuda.empty_cache()
                runs.append(dict(B=2, T=T, window=w, out_of_memory=oom, peak_GB=round(torch.cuda.max_memory_allocated() / 1e9, 2)))
            print(json.dumps(runs[-1]), flush=True)
    unet.set_temporal_window(None)
    res["runs"] = runs
    name, power = card()
    res.update(card=name, power_limit=power)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", default=None, help="default 25,49,64,96 (49,128 with --window)")
    ap.add_argument("--steps", type=int, default=5, help="timed DDIM steps per configuration")
    ap.add_argument("--warmup", type=int, default=2, help="untimed steps first (eager, capture)")
    ap.add_argument("--reps", type=int, default=200, help="temporal_attn launches per kernel timing")
    ap.add_argument("--window", default=None, help="W,S: measure windowed temporal attention instead")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_long_clip.py: no CUDA device")
    if args.window is not None:
        from viewcrafter_b200.temporal_window import check_window
        return window_main(args, check_window(tuple(int(v) for v in args.window.split(","))))
    import bench
    from bench_multicond import card

    torch.cuda.set_device(0)
    frames = sorted(int(t) for t in (args.frames or "25,49,64,96").split(","))
    res = {"metric": "long clips at 576x1024 (1 GPU, batch_cfg, graph replay)", "kernel": []}
    # kernel first, while the card holds nothing else of ours
    for sites, heads in ((H * W, 5), (H * W // 4, 10)):
        for T in (25, 49):
            res["kernel"].append(kernel_rate(2, T, sites, heads, args.reps))
    torch.cuda.empty_cache()
    model = bench.build_model(bench.WORKLOADS["ViewCrafter_25"], torch.device("cuda"))
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    budget = 0.9 * (free + torch.cuda.memory_allocated())
    res["budget_GB"] = round(budget / 1e9, 2)
    runs, fits, first2 = [], {}, None
    for B in (2, 3):
        pts = []
        for T in frames:
            if len(pts) >= 2:
                a, b = np.polyfit([p[0] for p in pts], [p[1] for p in pts], 1)
                pred = a * T + b
            elif pts:                                  # one point: proportional to T, an over-estimate (the weights do not grow)
                pred = pts[0][1] * T / pts[0][0]
            else:                                      # B = 3 before any of its points: B = 2's first peak times 3 / 2, in proportion
                pred = first2[1] * 1.5 * T / first2[0] if B == 3 and first2 else None
            if pred is not None and pred > budget:
                runs.append(dict(B=B, T=T, skipped=True, predicted_peak_GB=round(pred / 1e9, 2)))
                continue
            rate, peak, finite = time_steps(model, B, T, args.steps, args.warmup)
            pts.append((T, peak))
            runs.append(dict(B=B, T=T, steps_per_s=round(rate, 4), peak_GB=round(peak / 1e9, 2), finite=finite,
                             predicted_peak_GB=None if pred is None else round(pred / 1e9, 2)))
            print(json.dumps(runs[-1]), flush=True)
        if B == 2 and pts:
            first2 = pts[0]
        if len(pts) < 2:
            fits[f"B{B}"] = dict(skipped="fewer than two configurations fit")
            continue
        a, b = np.polyfit([p[0] for p in pts], [p[1] for p in pts], 1)
        resid = max(abs(a * t + b - p) / p for t, p in pts)
        t_mem = int((budget - b) // a)
        t_max = min(MAX_T, t_mem)
        entry = dict(GB_per_frame=round(a / 1e9, 4), GB_at_0=round(b / 1e9, 2), worst_linear_fit_residual=round(float(resid), 4),
                     memory_limit_T=t_mem, largest_T=t_max)
        if t_max >= 1:
            rate, peak, finite = time_steps(model, B, t_max, 1, 2)
            entry.update(confirm_steps_per_s=round(rate, 4), confirm_peak_GB=round(peak / 1e9, 2), confirm_finite=finite,
                         predicted_peak_GB=round((a * t_max + b) / 1e9, 2))
        fits[f"B{B}"] = entry
        print(json.dumps({f"B{B}": entry}), flush=True)
    res["runs"], res["largest_clip"] = runs, fits
    name, power = card()
    res.update(card=name, power_limit=power)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
