"""A/B micro-benchmark of the attention and GroupNorm kernels for side-by-side builds (VC_B200_LIB=<lib> python tools/ab_micro.py).
Prints the card and its power limit, then one line per kernel/shape: device ms (CUDA events, --reps launches after warm-up) and
max|err| vs a torch fp32 reference.

Bit-identity of two builds: run the first with --save DIR and the second with --compare DIR.  Both generate the same seeded
inputs; the attention outputs (self-attention l0 / l1 / l2, cross-attention Nk = 77 / 256 with accumulate) are written to DIR
and compared with torch.equal; the exit status is 1 if any differs."""
import argparse, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from viewcrafter_b200 import ops, _lib

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5, help="timed launches per shape")
ap.add_argument("--save", metavar="DIR", help="write the attention outputs to DIR")
ap.add_argument("--compare", metavar="DIR", help="compare the attention outputs with those --save wrote to DIR")
args = ap.parse_args()


def t(fn, reps=args.reps):
    fn(); fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3


mismatches = []


def keep(name, out):
    """Save or compare one attention output."""
    if args.save:
        os.makedirs(args.save, exist_ok=True)
        torch.save(out.cpu(), os.path.join(args.save, name + ".pt"))
    if args.compare:
        ref = torch.load(os.path.join(args.compare, name + ".pt")).to(out.device)
        same = torch.equal(out, ref)
        if not same:
            mismatches.append(name)
        print(f"[{tag}]   {name}: " + ("bit-identical" if same else f"DIFFERS, max |diff| {float((out.float() - ref.float()).abs().max()):.3e}"))


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


tag = os.path.basename(_lib.LIB_PATH) + ("+bn64" if os.environ.get("VC_ATTN_BN64") == "1" else "")
print(f"[{tag}] {torch.cuda.get_device_name()}, power limit {power_limit()}")
T = 25
torch.manual_seed(0)
for name, HW, heads in (("l0", 9216, 5), ("l1", 2304, 10), ("l2", 576, 20)):
    C = heads * 64
    qkv = (torch.randn(T * HW, 3 * C, device="cuda") * 0.7).half()
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    dt = t(lambda: ops.flash_attn(q, k, v, T, HW, HW, heads))
    fl = 4.0 * T * heads * HW * HW * 64
    qq, kk, vv = (x[:HW, 64:128].float() for x in (q, k, v))
    ref = torch.softmax(qq @ kk.t() * 0.125, -1) @ vv
    full = ops.flash_attn(q, k, v, T, HW, HW, heads)
    out = full[:HW, 64:128].float()
    print(f"[{tag}] self-attn {name} N={HW:5d} heads={heads:2d}: {dt*1e3:7.3f} ms {fl/dt/1e12:7.1f} TFLOP/s  max err {float((out-ref).abs().max()):.2e}")
    keep(f"self_{name}", full)
kv = (torch.randn(333, 2 * 320, device="cuda") * 0.7).half()
q = (torch.randn(T * 9216, 320, device="cuda") * 0.7).half()
base = (torch.randn(T * 9216, 320, device="cuda") * 0.5).half()
for Nk in (77, 256):
    dt = t(lambda: ops.flash_attn(q, kv[:Nk, :320], kv[:Nk, 320:], T, 9216, Nk, 5, kv_shared=True))
    acc = base.clone()
    dta = t(lambda: ops.flash_attn(q, kv[:Nk, :320], kv[:Nk, 320:], T, 9216, Nk, 5, kv_shared=True, out=acc, accumulate=True))
    print(f"[{tag}] cross-attn l0 Nk={Nk:3d}: {dt*1e6:8.1f} us, with accumulate {dta*1e6:8.1f} us")
    acc = base.clone()
    ops.flash_attn(q, kv[:Nk, :320], kv[:Nk, 320:], T, 9216, Nk, 5, kv_shared=True, out=acc, accumulate=True)
    keep(f"cross_{Nk}_acc", acc)
for name, H, W, C, samples in (("l0 4-D", 72, 128, 320, 25), ("l0 4-D B=2", 72, 128, 320, 50), ("l1 4-D", 36, 64, 640, 25), ("l2 4-D", 18, 32, 1280, 25),
                               ("l1 5-D", 36, 64, 640, 1), ("l2 5-D", 18, 32, 1280, 1)):
    M = T * H * W * (2 if samples == 50 else 1)
    x = (torch.randn(M, C, device="cuda") * 0.8 + 0.1).half()
    g, b = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.1
    dt = t(lambda: ops.groupnorm(x, samples, g, b, 1e-5, True))
    y = ops.groupnorm(x, samples, g, b, 1e-5, True).float()
    xr = x.float().reshape(samples, -1, 32, C // 32)
    mu = xr.mean((1, 3), keepdim=True); var = xr.var((1, 3), unbiased=False, keepdim=True)
    ref = ((xr - mu) * torch.rsqrt(var + 1e-5)).reshape(M, C) * g + b
    ref = ref * torch.sigmoid(ref)
    print(f"[{tag}] groupnorm {name:10s} C={C:4d}: {dt*1e6:8.1f} us  {2.0*M*C*2/dt/1e9:7.1f} GB/s (r+w once)  max err {float((y-ref).abs().max()):.2e}")
for name, M, C in (("l0", 230400, 320), ("l1", 57600, 640), ("l2", 14400, 1280), ("init", 230400, 512)):
    x = (torch.randn(M, C, device="cuda") * 0.8 + 0.3).half()
    dt = t(lambda: ops.layernorm_stats(x))
    st = ops.layernorm_stats(x)
    xf = x.float()
    ref_mean, ref_rstd = xf.mean(1), torch.rsqrt(xf.var(1, unbiased=False) + 1e-5)
    err = max(float((st[:, 0] - ref_mean).abs().max()), float(((st[:, 1] - ref_rstd) / ref_rstd).abs().max()))
    print(f"[{tag}] ln_stats {name:4s} C={C:4d}: {dt*1e6:8.1f} us  {M*C*2/dt/1e9:7.1f} GB/s  max err {err:.2e}")
if args.compare:
    print(f"[{tag}] outputs vs {args.compare}: " + (f"DIFFER: {', '.join(mismatches)}" if mismatches else "all bit-identical"))
    sys.exit(1 if mismatches else 0)
