#!/usr/bin/env python
"""Seconds per image_guided_synthesis call and per output at 576x1024 x 25 frames, for every replica count R that divides the world
(parallel.shard_model(replicas=R)) and n_samples in --n-samples.

    python -m torch.distributed.run --nproc-per-node N tools/bench_replicas.py
    python tools/bench_replicas.py                      # one GPU: R = 1 only

The model is bench.py's random-weight full-width U-Net plus a random-init full-width VAE, perframe_ae=True; one clip (B=1), two-way
guidance (CFG 7.5, rescale 0.7, eta 1), batch_cfg and graph replay; stand-ins for the image embedder, its projection and the text
encoder produce the 333-token context.  A call is encode + sampling + decode, timed with the host clock from a barrier to a device
synchronise and a barrier, the slowest rank's time.  Every layout is created once and runs one untimed call of each n_samples first.
Then, --repeats times, each R > 1 is timed right after an R = 1 run (R = 1 runs alternate with R > 1 runs); medians are reported,
with the largest difference of each R's output from R = 1's (same seed).  Prints one JSON line with the card name and its power limit.
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=50, help="DDIM steps per sample")
    ap.add_argument("--n-samples", default="1,2,4,8", help="n_samples values to time")
    ap.add_argument("--repeats", type=int, default=1, help="timed runs of every (n_samples, R); medians are reported")
    args = ap.parse_args()
    import bench
    from bench_multicond import card
    from viewcrafter_b200 import parallel
    from viewcrafter_b200.autoencoder import AutoencoderKL
    from viewcrafter_b200.configs import VAE_DDCONFIG
    from viewcrafter_b200.synthesis import image_guided_synthesis

    if not torch.cuda.is_available():
        raise SystemExit("bench_replicas.py: no CUDA device")
    world, rank, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    wl = bench.WORKLOADS["ViewCrafter_25"]
    model = bench.build_model(wl, device).to(device)            # the schedule buffers too: the sampler draws x_T on their device
    torch.manual_seed(3)
    with torch.device(device):
        model.first_stage_model = AutoencoderKL(VAE_DDCONFIG, None, 4).eval()
    g = torch.Generator().manual_seed(4)
    W_img = (torch.randn(3 * 4 * 4, 256 * 1024, generator=g) * 0.01).to(device)
    txt, txt_empty = torch.randn(1, 77, 1024, generator=g).to(device), torch.randn(1, 77, 1024, generator=g).to(device)
    model.embedder = lambda img: torch.nn.functional.adaptive_avg_pool2d(img, 4).reshape(img.shape[0], 1, -1)
    model.image_proj_model = lambda e: (e @ W_img).reshape(e.shape[0], 256, 1024)
    model.get_learned_conditioning = lambda prompts: torch.cat([txt_empty if p == "" else txt for p in prompts], 0)
    model.uncond_type = "empty_seq"
    T, h, w = wl["T"], wl["H"], wl["W"]
    videos = (torch.rand(1, 3, T, 8 * h, 8 * w, generator=g) * 2 - 1).to(device)

    # every layout once (shard_model creates process groups and peer buffers); switching layouts then only swaps the attributes
    unet = model.model.diffusion_model
    Rs = [r for r in range(1, world + 1) if world % r == 0]
    layouts = {}
    for R in Rs:
        if world > 1:
            model.__dict__.pop("_cfg", None)
            model.__dict__.pop("_replicas", None)
            parallel.shard_model(model, dist, rank, world, replicas=R)
        layouts[R] = (model.__dict__.get("_cfg"), model.__dict__.get("_replicas"), unet._comm)

    def use(R):
        cfg, reps, comm = layouts[R]
        model.__dict__.pop("_cfg", None)
        model.__dict__.pop("_replicas", None)
        if cfg is not None:
            model._cfg = cfg
        if reps is not None:
            model._replicas = reps
        unet._comm = comm

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    def call(R, n):
        use(R)
        barrier()
        t0 = time.perf_counter()
        torch.manual_seed(5)
        out = image_guided_synthesis(model, ["a photo"], videos, [1, 4, T, h, w], n_samples=n, ddim_steps=args.steps, ddim_eta=1.0,
                                     unconditional_guidance_scale=7.5, fs=10, text_input=True, timestep_spacing="uniform_trailing",
                                     guidance_rescale=0.7, condition_index=[0])
        barrier()
        dt = torch.tensor([time.perf_counter() - t0], device=device, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(dt, op=dist.ReduceOp.MAX)                # the slowest rank sets the pace
        return out, float(dt)

    ns = [int(v) for v in args.n_samples.split(",") if v]
    for n in ns:                                                     # warm-up: every layout and shape once (graph capture)
        for R in Rs:
            call(R, n)
    times = {(n, R): [] for n in ns for R in Rs}
    diffs = {}
    for _ in range(args.repeats):
        for n in ns:
            for R in (Rs[1:] or [None]):
                ref, t = call(1, n)
                times[(n, 1)].append(t)
                if R is not None:
                    out, t = call(R, n)
                    times[(n, R)].append(t)
                    diffs[(n, R)] = max(diffs.get((n, R), 0.0), float((out - ref).abs().max()))
    name, power = card()
    if rank == 0:
        res = []
        for (n, R), v in times.items():
            s = float(np.median(v))
            res.append({"n_samples": n, "replicas": R, "gpus_per_group": world // R, "s_per_call": s, "s_per_output": s / n, "runs": v,
                        "max_abs_diff_vs_R1": diffs.get((n, R), 0.0 if R == 1 else None)})
        print(json.dumps({"metric": "seconds per image_guided_synthesis call", "workload": "ViewCrafter_25", "px": wl["px"], "frames": T,
                          "gpus": world, "clips": 1, "ddim_steps": args.steps, "perframe_ae": model.perframe_ae, "results": res,
                          "card": name, "power_limit": power}), flush=True)
    bench._finish(world, dist)


if __name__ == "__main__":
    main()
