"""FP8 mode against fp16 on one GPU: DDIM steps/s at 576x1024x25 with two-way CFG (one B=2 forward per step, CUDA graph), three
alternating runs of each mode; fp16 and fp8 TFLOP/s of the tap-GEMM shape classes of that forward, the fp8 GEMM timed alone with a
precomputed activation amax and the absmax pass timed separately; the absmax kernel's share of the kernel time of one fp8 forward
(torch.profiler).  Prints one JSON line with the card name and its power limit.

    python tools/bench_fp8.py [--steps 10] [--repeats 3] [--parity path/to/parity_fp8.json]

--parity adds the accuracy numbers tests/test_fp8_unet_gpu.py wrote (VC_PARITY_OUT) to the output.
"""
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


def gemm_classes(ops, T=25):
    """(name, flop, fp16 call, fp8 GEMM call with a precomputed amax, absmax call) for the GEMM shape classes of a 25x72x128
    forward (B=2 rows)."""
    dev = "cuda"
    rnd = lambda *s: (torch.randn(*s, device=dev) * 0.05).half()
    out = []

    def gemm_only(call, x, w8, amax):
        real = ops.absmax
        ops.absmax = lambda *a, **k: amax              # the GEMM alone: the activation scale is already known
        try:
            return call(x, w8)
        finally:
            ops.absmax = real

    def add(name, flop, x, w16, taps, call):
        w8 = ops.Fp8Weight(*ops.pack_fp8(w16, taps))
        amax = ops.absmax(x)
        out.append((name, flop, lambda: call(x, w16), lambda: gemm_only(call, x, w8, amax), lambda: ops.absmax(x, out=amax)))

    B = 2
    for H, W, C, lv in ((72, 128, 320, 0), (36, 64, 640, 1), (18, 32, 1280, 2)):
        M = B * T * H * W
        x, r = rnd(M, C), rnd(M, C)
        b = torch.zeros(C, device=dev)
        add(f"conv3x3 l{lv} {C}->{C} +res", 2.0 * M * 9 * C * C, x, rnd(9 * C, C), 9,
            lambda x, w, H=H, W=W, b=b, r=r: ops.conv3x3(x, B * T, H, W, w, bias=b, res=r))
        add(f"tconv l{lv} {C}", 2.0 * M * 3 * C * C, x, rnd(3 * C, C), 3, lambda x, w, H=H, W=W, b=b: ops.conv_temporal(x, B, T, H * W, w, bias=b))
        add(f"linear l{lv} {C}->{C} +res", 2.0 * M * C * C, x, rnd(C, C), 1, lambda x, w, b=b, r=r: ops.linear(x, w, bias=b, res=r))
        add(f"qkv l{lv} {C}->{3 * C}", 2.0 * M * C * 3 * C, x, rnd(3 * C, C), 1, lambda x, w: ops.linear(x, w))
        wg, bg = ops.pack_geglu(rnd(8 * C, C), torch.zeros(8 * C, device=dev))
        add(f"geglu l{lv} {C}->{8 * C}", 2.0 * M * C * 8 * C, x, wg, 1, lambda x, w, bg=bg: ops.linear(x, w, bias=bg, geglu=True))
        x4 = rnd(M, 4 * C)
        add(f"ff2 l{lv} {4 * C}->{C} +res", 2.0 * M * 4 * C * C, x4, rnd(C, 4 * C), 1, lambda x, w, b=b, r=r: ops.linear(x, w, bias=b, res=r))
    return out


def event_time(fn, reps=10):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--parity", default=None)
    args = ap.parse_args()
    import bench
    from bench_multicond import card
    from viewcrafter_b200 import ops
    from viewcrafter_b200.ddim import DDIMSampler

    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8.py: no CUDA device")
    device = torch.device("cuda", 0)
    wl = bench.WORKLOADS["ViewCrafter_25"]
    model = bench.build_model(wl, device)
    unet = model.model.diffusion_model
    unet.enable_cuda_graph()
    _, dev = bench.synthetic_inputs(wl, device)
    T, h, w = wl["T"], wl["H"], wl["W"]
    fs = torch.tensor([10], device=device, dtype=torch.long)
    lat = torch.randn(1, 4, T, h, w, generator=torch.Generator().manual_seed(4)).to(device)

    def sample(steps):
        c = {"c_crossattn": [dev["ctx_c"]], "c_concat": [lat]}
        uc = {"c_crossattn": [dev["ctx_u"]], "c_concat": [lat]}
        out, _ = DDIMSampler(model, batch_cfg=True).sample(S=steps, batch_size=1, shape=(4, T, h, w), conditioning=c, verbose=False,
                                                           unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=1.0,
                                                           fs=fs, timestep_spacing="uniform_trailing", guidance_rescale=0.7, x_T=dev["x_T"])
        return out

    rates = {"fp16": [], "fp8": []}
    for mode in ("fp16", "fp8"):                     # warm-up: packs, K/V cache, graph capture of each mode
        unet.enable_fp8(mode == "fp8")
        sample(3)
    for _ in range(args.repeats):
        for mode in ("fp16", "fp8"):
            unet.enable_fp8(mode == "fp8")
            torch.manual_seed(5)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = sample(args.steps)
            torch.cuda.synchronize()
            rates[mode].append(args.steps / (time.perf_counter() - t0))
            assert torch.isfinite(out).all(), mode

    # absmax share of one fp8 forward's kernel time (eager, B=2)
    unet.enable_cuda_graph(False)
    unet.enable_fp8(True)
    xb = torch.cat([torch.cat([dev["x_T"], lat], 1)] * 2)
    ctx = torch.cat([dev["ctx_c"], dev["ctx_u"]])
    tt = torch.full((2,), 999, device=device, dtype=torch.long)
    fwd = lambda: unet(xb, tt, context=ctx, fs=fs.repeat(2), cfg_shared_prefix=True)
    fwd()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fwd()
        torch.cuda.synchronize()
    tot = absm = 0.0
    for e in prof.key_averages():
        dt = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if e.key.startswith(("gemm_", "void vc::", "vc::")) or "kernel" in e.key:
            tot += dt
            if "absmax" in e.key:
                absm += dt
    unet.enable_fp8(False)

    gemms = []
    for name, flop, f16, f8, am in gemm_classes(ops):
        t16, t8, ta = event_time(f16), event_time(f8), event_time(am)
        gemms.append({"shape": name, "fp16_tflops": flop / t16 / 1e12, "fp8_gemm_tflops": flop / t8 / 1e12, "fp16_us": t16 * 1e6,
                      "fp8_gemm_us": t8 * 1e6, "absmax_us": ta * 1e6})
    med = lambda v: float(np.median(v))
    parity = None
    if args.parity and os.path.exists(args.parity):
        parity = json.load(open(args.parity))
    name, power = card()
    print(json.dumps({"metric": "fp8 vs fp16 DDIM steps/s", "workload": "ViewCrafter_25", "px": wl["px"], "frames": T, "cfg": "two-way, B=2",
                      "steps": args.steps, "fp16_steps_per_s": med(rates["fp16"]), "fp8_steps_per_s": med(rates["fp8"]),
                      "fp16_runs": rates["fp16"], "fp8_runs": rates["fp8"], "speedup": med(rates["fp8"]) / med(rates["fp16"]),
                      "absmax_share_of_fp8_forward_kernel_time": absm / tot if tot else None, "gemm_classes": gemms,
                      "accuracy": parity, "card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
