#!/usr/bin/env python
"""DPM-Solver++(2M) and (3M) SDE against DDIM on the full-width U-Net at 576x1024 x 25 frames, one GPU.

    python tools/bench_dpm.py [--dpm-steps 15,20,25] [--dpm3-steps 8,10,15] [--ode-steps 10,20,25,50] [--ode-ref-steps 200]

1. Seconds per clip, sampling + VAE decode: DDIM at --ddim-steps (50, the ViewCrafter default), DPM-Solver++(2M) at each of
   --dpm-steps and DPM-Solver++(3M) SDE at each of --dpm3-steps.  All run ViewCrafter's sampling settings: two-way CFG 7.5, guidance
   rescale 0.7, eta 1, uniform_trailing, batch_cfg and graph replay.  Host clock around work that ends in a device synchronise, after
   one untimed warm-up of every stage.
2. The ODE convergence of the real U-Net (eta 0, same guidance): the error of DDIM and DPM-Solver++(2M) at each of --ode-steps against
   a DPM-Solver++(2M) run of --ode-ref-steps from the same x_T, as max |diff| and RMS / RMS of the reference.

The weights are bench.py's random full-width U-Net and a random-init full-width VAE, so the numbers say how the solvers converge on
this network and what a step costs, not what a clip looks like on the released checkpoint.  Prints one JSON line with the card name
and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--ddim-steps", type=int, default=50)
    ap.add_argument("--dpm-steps", default="15,20,25")
    ap.add_argument("--dpm3-steps", default="8,10,15")
    ap.add_argument("--ode-steps", default="10,20,25,50", help="empty: skip the convergence table")
    ap.add_argument("--ode-ref-steps", type=int, default=200)
    args = ap.parse_args()
    import bench
    from bench_multicond import card
    from viewcrafter_b200.autoencoder import AutoencoderKL
    from viewcrafter_b200.configs import VAE_DDCONFIG
    from viewcrafter_b200.ddim import DDIMSampler
    from viewcrafter_b200.dpm_solver import DPMSolver3MSDESampler, DPMSolverSampler

    if not torch.cuda.is_available():
        raise SystemExit("bench_dpm.py: no CUDA device")
    device = torch.device("cuda", 0)
    wl = bench.WORKLOADS["ViewCrafter_25"]
    model = bench.build_model(wl, device)
    torch.manual_seed(3)
    with torch.device(device):
        model.first_stage_model = AutoencoderKL(VAE_DDCONFIG, None, 4).eval()
    model.model.diffusion_model.enable_cuda_graph()
    _, dev = bench.synthetic_inputs(wl, device)
    T, h, w = wl["T"], wl["H"], wl["W"]
    fs = torch.tensor([10], device=device, dtype=torch.long)
    c = {"c_crossattn": [dev["ctx_c"]], "c_concat": [dev["c_concat"]]}
    uc = {"c_crossattn": [dev["ctx_u"]], "c_concat": [dev["c_concat"]]}

    def sample(cls, steps, eta, x_T):
        out, _ = cls(model, batch_cfg=True).sample(S=steps, batch_size=1, shape=(4, T, h, w), conditioning=c, verbose=False,
                                                   unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=eta, fs=fs,
                                                   timestep_spacing="uniform_trailing", guidance_rescale=0.7, x_T=x_T)
        return out

    def clip(cls, steps):
        torch.manual_seed(7)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        z = sample(cls, steps, 1.0, dev["x_T"])
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        y = model.decode_first_stage(z)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        assert bool(torch.isfinite(y).all())
        return {"sampling_s": t1 - t0, "decode_s": t2 - t1, "clip_s": t2 - t0, "s_per_step": (t1 - t0) / steps}

    # warm-up: both samplers (the third forward captures the U-Net's graph) and the decode
    torch.manual_seed(5)
    model.decode_first_stage(sample(DDIMSampler, 3, 1.0, dev["x_T"]))
    sample(DPMSolverSampler, 5, 1.0, dev["x_T"])
    sample(DPMSolver3MSDESampler, 5, 1.0, dev["x_T"])
    timing = {f"ddim_{args.ddim_steps}": clip(DDIMSampler, args.ddim_steps)}
    for s in [int(v) for v in args.dpm_steps.split(",") if v]:
        timing[f"dpmpp_2m_{s}"] = clip(DPMSolverSampler, s)
    for s in [int(v) for v in args.dpm3_steps.split(",") if v]:
        timing[f"dpmpp_3m_sde_{s}"] = clip(DPMSolver3MSDESampler, s)

    ode = {}
    ode_steps = [int(v) for v in args.ode_steps.split(",") if v]
    if ode_steps:
        x_T = dev["x_T"]
        ref = sample(DPMSolverSampler, args.ode_ref_steps, 0.0, x_T).double()
        rms = lambda t: float(t.pow(2).mean().sqrt())
        for s in ode_steps:
            for name, cls in (("ddim", DDIMSampler), ("dpmpp_2m", DPMSolverSampler)):
                d = sample(cls, s, 0.0, x_T).double() - ref
                ode[f"{name}_{s}"] = {"max_abs": float(d.abs().max()), "rel_rms": rms(d) / rms(ref)}
    name, power = card()
    print(json.dumps({"metric": "DPM-Solver++(2M) / (3M) SDE vs DDIM", "workload": "ViewCrafter_25", "px": wl["px"], "frames": T,
                      "settings": "CFG 7.5, guidance rescale 0.7, uniform_trailing, batch_cfg, graph replay; clip timing eta 1, ODE eta 0",
                      "seconds_per_clip": timing, "ode_reference": f"dpmpp_2m_{args.ode_ref_steps} from the same x_T", "ode_error": ode,
                      "card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
