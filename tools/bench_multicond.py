#!/usr/bin/env python
"""Three-way classifier-free guidance throughput: DDIM steps/s of ddim_multiplecond.DDIMSampler at 576x1024 x 25 frames.

    python tools/bench_multicond.py --steps 10 --warmup 3 --repeats 3
    python -m torch.distributed.run --nproc-per-node N tools/bench_multicond.py --layout cfg_split   # or --layout frames

One step = one p_sample_ddim with CFG 7.5, cfg_img 2.0, guidance rescale 0.7, eta 1: three U-Net predictions (cond, uncond,
uncond_img) and the fused three-way update.  The model is bench.py's random-weight full-width U-Net with synthetic inputs, the
forward is replayed as a CUDA graph (--no-graph: eager), and time is measured with CUDA events: `repeats` windows of `steps`
steps after `warmup` steps, each window ending in a synchronise of all ranks; the median window gives the rate.
Layouts on N GPUs: cfg_split = ranks 0..N/2-1 compute cond, the rest uncond + uncond_img (one B=2 forward), each half
frame-sharded N/2 ways; frames = one B=3 forward frame-sharded over all N ranks.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """Name and power limit of the current GPU as nvidia-smi reports them."""
    idx = torch.cuda.current_device()
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(idx), "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10, help="steps per timed window")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3, help="timed windows; the median is reported")
    ap.add_argument("--workload", default="ViewCrafter_25")
    ap.add_argument("--layout", choices=["cfg_split", "frames"], default="cfg_split", help="multi-GPU layout (ignored on one GPU)")
    ap.add_argument("--no-batch-cfg", action="store_true", help="three separate forwards per step")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--dump-outputs", default=None, help="write the last timed step's x_prev / pred_x0 as DIR/<name>.npy")
    args = ap.parse_args()
    import bench
    from viewcrafter_b200.ddim_multiplecond import DDIMSampler

    if not torch.cuda.is_available():
        raise SystemExit("bench_multicond.py: no CUDA device")
    world, rank, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    wl = bench.WORKLOADS[args.workload]
    model = bench.build_model(wl, device)
    layout = "1 GPU"
    if world > 1:
        from viewcrafter_b200 import parallel
        parallel.shard_model(model, dist, rank, world, cfg_split=args.layout == "cfg_split")
        layout = args.layout
    unet = model.model.diffusion_model
    if not args.no_graph:
        unet.enable_cuda_graph()
    sampler = DDIMSampler(model, batch_cfg=not args.no_batch_cfg)
    sampler.make_schedule(50, "uniform_trailing", 1.0, verbose=False)
    _, dev = bench.synthetic_inputs(wl, device)
    c, uc = bench.conds(dev, None)
    ctx_i = torch.randn(1, 333, 1024, generator=torch.Generator().manual_seed(5)).to(device)
    ui = {"c_crossattn": [ctx_i], "c_concat": [dev["c_concat"]]}
    fs = torch.tensor([10], device=device, dtype=torch.long)
    order = np.flip(sampler.ddim_timesteps)

    def run_step(x, i):
        i = i % 50
        ts = torch.full((1,), int(order[i]), device=device, dtype=torch.long)
        return sampler.p_sample_ddim(x, c, ts, index=50 - i - 1, unconditional_guidance_scale=7.5, unconditional_conditioning=uc,
                                     cfg_img=2.0, unconditional_conditioning_img_nonetext=ui, fs=fs, guidance_rescale=0.7,
                                     _step=int(order[i]))

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    torch.manual_seed(0)
    x = dev["x_T"]
    for i in range(args.warmup):
        x, _ = run_step(x, i)
    barrier()
    rates, k = [], args.warmup
    for _ in range(args.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            x, pred_x0 = run_step(x, k)
            k += 1
        e1.record()
        barrier()
        dt = torch.tensor([e0.elapsed_time(e1) * 1e-3], device=device, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(dt, op=dist.ReduceOp.MAX)                # the slowest rank sets the pace
        rates.append(args.steps / float(dt))
    if args.dump_outputs and rank == 0:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, t in (("x_prev", x), ("pred_x0", pred_x0)):
            np.save(os.path.join(args.dump_outputs, name + ".npy"), t.detach().float().cpu().numpy())
    name, power = card()
    if rank == 0:
        print(json.dumps({"metric": "three-way CFG DDIM steps/s", "workload": args.workload, "px": wl["px"], "frames": wl["T"],
                          "gpus": world, "layout": layout, "batch_cfg": not args.no_batch_cfg, "graph": not args.no_graph,
                          "steps_per_s": float(np.median(rates)), "windows": [round(r, 4) for r in rates],
                          "steps_per_window": args.steps, "warmup": args.warmup, "finite": bool(torch.isfinite(x).all()),
                          "card": name, "power_limit": power}), flush=True)
    bench._finish(world, dist)


if __name__ == "__main__":
    main()
