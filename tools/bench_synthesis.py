#!/usr/bin/env python
"""Stage wall-clock of one ViewCrafter_25 clip at 576x1024 x 25 frames: VAE encode of the 25 conditioning renders
(synthesis.get_latent_z), 50-step two-way DDIM sampling, VAE decode of the 25 output frames.

    python tools/bench_synthesis.py
    python -m torch.distributed.run --nproc-per-node N tools/bench_synthesis.py

The model is bench.py's random-weight full-width U-Net plus a random-init full-width VAE, perframe_ae=True (the ViewCrafter
default); sampling runs CFG 7.5, guidance rescale 0.7, eta 1, with batch_cfg and graph replay.  Under torchrun shard_model picks
its default layout (CFG split for an even world) and the VAE is frame-sharded over all ranks.  Each time is the host clock around
work that ends in a device synchronise (and a barrier of all ranks), after one untimed run of every stage.  The sharded VAE
(parallel.vae_encode / vae_decode) and the unsharded calls every rank would otherwise make (get_latent_z's encode_first_stage,
decode_first_stage) alternate, --repeats times each; the medians are reported, with the all-gather of the decoded frames timed on
its own.  On one GPU the two are the same calls; there it also times the largest share of 2, 4 and 8 ranks (rank 0's frames:
the per-rank VAE work, without the all-gather).  Prints one JSON line with the card name and its power limit.
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
    ap.add_argument("--steps", type=int, default=50, help="DDIM steps of the clip")
    ap.add_argument("--repeats", type=int, default=3, help="timed runs of each VAE variant (alternating); the medians are reported")
    ap.add_argument("--share-worlds", default="2,4,8",
                    help="on one GPU: also time the largest VAE share (rank 0's frames) of these world sizes, without the gather")
    args = ap.parse_args()
    import bench
    from bench_multicond import card
    from viewcrafter_b200 import parallel
    from viewcrafter_b200.autoencoder import AutoencoderKL
    from viewcrafter_b200.configs import VAE_DDCONFIG
    from viewcrafter_b200.ddim import DDIMSampler
    from viewcrafter_b200.synthesis import get_latent_z

    if not torch.cuda.is_available():
        raise SystemExit("bench_synthesis.py: no CUDA device")
    world, rank, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    wl = bench.WORKLOADS["ViewCrafter_25"]
    model = bench.build_model(wl, device)
    torch.manual_seed(3)
    with torch.device(device):
        model.first_stage_model = AutoencoderKL(VAE_DDCONFIG, None, 4).eval()
    layout = "1 GPU"
    if world > 1:
        parallel.shard_model(model, dist, rank, world)
        layout = "cfg_split" if world % 2 == 0 else "frames"
    vae_comm = getattr(model, "_vae_comm", None)
    model.model.diffusion_model.enable_cuda_graph()
    _, dev = bench.synthetic_inputs(wl, device)
    T, h, w = wl["T"], wl["H"], wl["W"]
    videos = (torch.rand(1, 3, T, 8 * h, 8 * w, generator=torch.Generator().manual_seed(4)) * 2 - 1).to(device)
    fs = torch.tensor([10], device=device, dtype=torch.long)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    def timed(fn):
        barrier()
        t0 = time.perf_counter()
        out = fn()
        barrier()
        dt = torch.tensor([time.perf_counter() - t0], device=device, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(dt, op=dist.ReduceOp.MAX)                # the slowest rank sets the pace
        return out, float(dt)

    def unsharded(fn):
        model._vae_comm = None
        try:
            return fn()
        finally:
            model._vae_comm = vae_comm

    encode = lambda: get_latent_z(model, videos)
    decode = lambda zz: parallel.vae_decode(model, zz) if vae_comm else model.decode_first_stage(zz)

    def sample(latents, steps):
        c = {"c_crossattn": [dev["ctx_c"]], "c_concat": [latents]}
        uc = {"c_crossattn": [dev["ctx_u"]], "c_concat": [latents]}
        out, _ = DDIMSampler(model, batch_cfg=True).sample(S=steps, batch_size=1, shape=(4, T, h, w), conditioning=c, verbose=False,
                                                           unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=1.0,
                                                           fs=fs, timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                                                           x_T=dev["x_T"])
        return out

    # warm-up: every stage once (the sampler's third forward captures the U-Net's CUDA graph)
    torch.manual_seed(5)
    latents = encode()
    unsharded(encode)
    samples = sample(latents, 3)
    decode(samples)
    unsharded(lambda: model.decode_first_stage(samples))

    samples, t_sample = timed(lambda: sample(latents, args.steps))
    enc_s, enc_u, dec_s, dec_u, gather = [], [], [], [], []
    share_worlds = [int(p) for p in args.share_worlds.split(",") if p] if world == 1 else []
    shares = {P: {"encode": [], "decode": []} for P in share_worlds}
    for _ in range(args.repeats):
        enc_s.append(timed(encode)[1])
        enc_u.append(timed(lambda: unsharded(encode))[1])
        y_s, t = timed(lambda: decode(samples))
        dec_s.append(t)
        y_u, t = timed(lambda: unsharded(lambda: model.decode_first_stage(samples)))
        dec_u.append(t)
        if vae_comm:
            share = parallel.vae_decode_share(model, samples, vae_comm.rank, vae_comm.world)
            gather.append(timed(lambda: parallel.gather_shares(vae_comm, share, T, device, samples.dtype))[1])
        # the work of the largest share (rank 0's) of every world size in --share-worlds, on this GPU alone: no gather
        for P in share_worlds:
            shares[P]["encode"].append(timed(lambda: parallel.vae_encode_share(model, videos, 0, P))[1])
            shares[P]["decode"].append(timed(lambda: parallel.vae_decode_share(model, samples, 0, P))[1])
    same = bool(torch.equal(y_s, y_u))
    med = lambda v: float(np.median(v)) if v else None
    name, power = card()
    if rank == 0:
        clip_s = med(enc_s) + t_sample + med(dec_s)
        clip_u = med(enc_u) + t_sample + med(dec_u)
        print(json.dumps({"metric": "seconds per clip by stage", "workload": "ViewCrafter_25", "px": wl["px"], "frames": T, "gpus": world,
                          "layout": layout, "ddim_steps": args.steps, "perframe_ae": model.perframe_ae,
                          "encode_s_sharded": med(enc_s), "encode_s_unsharded": med(enc_u),
                          "decode_s_sharded": med(dec_s), "decode_s_unsharded": med(dec_u), "decode_gather_s": med(gather),
                          "sampling_s": t_sample, "clip_s_sharded_vae": clip_s, "clip_s_unsharded_vae": clip_u,
                          "runs": {"encode_sharded": enc_s, "encode_unsharded": enc_u, "decode_sharded": dec_s, "decode_unsharded": dec_u,
                                   "gather": gather},
                          "largest_share_s_one_gpu": {P: {"frames": parallel.frame_ranges(T, P)[0][1], "encode_s": med(v["encode"]),
                                                          "decode_s": med(v["decode"])} for P, v in shares.items()},
                          "decoded_bit_identical": same, "finite": bool(torch.isfinite(y_s).all()),
                          "card": name, "power_limit": power}), flush=True)
    bench._finish(world, dist)


if __name__ == "__main__":
    main()
