"""Micro-benchmark of the tap-GEMM on the shapes that dominate a 25x72x128 U-Net forward (development tool).

Rows are B * 25 frames: the batched classifier-free-guidance forward of bench.py runs B = 2.  Every transformer class is timed
as the U-Net calls it: qkv and GEGLU with the LayerNorm folded in, the C->C `in` projection leaving LayerNorm statistics
(ln_out), the `out` projection adding the residual and leaving GroupNorm statistics (gn_out).  Each time includes the small
statistics-finishing kernels of ln_out / gn_out.  --json prints one JSON object (for A/B runs: VC_B200_LIB selects the build).
"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from viewcrafter_b200 import ops

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=2, help="samples per forward (rows = batch * 25 frames * H * W)")
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--json", action="store_true")
args = ap.parse_args()

dev = "cuda"
def t(fn, reps=args.reps):
    fn(); fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3

def rnd(*s): return (torch.randn(*s, device=dev) * 0.05).half()
T = 25 * args.batch
rows = []
def add(name, flop, dt, nbytes=None):
    rows.append({"name": name, "tflops": flop / dt / 1e12, "us": dt * 1e6, "gbs": None if nbytes is None else nbytes / dt / 1e9})
def lin(name, M, K, N, res=False, geglu=False, bias=True, ln=False, ln_out=False, gn_out=False):
    x, w = rnd(M, K), rnd(N, K)
    b = torch.zeros(N, device=dev) if bias else None
    if geglu: w, b = ops.pack_geglu(w, b)
    r = rnd(M, N) if res else None
    lnarg = (ops.layernorm_stats(x), w.float().sum(1).contiguous()) if ln else None
    dt = t(lambda: ops.linear(x, w, bias=b, res=r, geglu=geglu, ln=lnarg, ln_out=ln_out, gn_out=gn_out))
    n_out = N // 2 if geglu else N
    add(name, 2.0 * M * K * N, dt, 2.0 * M * (K + n_out + (N if res else 0)))   # HBM floor: read A (+ residual), write out
def conv(name, H, W, Ci, Co, res=False):
    x, w9 = rnd(T * H * W, Ci), rnd(9 * Co, Ci)
    b = torch.zeros(Co, device=dev); r = rnd(T * H * W, Co) if res else None
    dt = t(lambda: ops.conv3x3(x, T, H, W, w9, bias=b, res=r))
    add(name, 2.0 * T * H * W * 9 * Ci * Co, dt)
def tconv(name, HW, C):
    x, w3 = rnd(T * HW, C), rnd(3 * C, C)
    b = torch.zeros(C, device=dev)
    dt = t(lambda: ops.conv_temporal(x, 1, T, HW, w3, bias=b))
    add(name, 2.0 * T * HW * 3 * C * C, dt)

M0, M1, M2, M3 = T * 9216, T * 2304, T * 576, T * 144
conv("conv3x3 l0 320->320 +res", 72, 128, 320, 320, res=True)
conv("conv3x3 l0 960->320", 72, 128, 960, 320)
conv("conv3x3 l1 640->640 +res", 36, 64, 640, 640, res=True)
conv("conv3x3 l2 1280->1280 +res", 18, 32, 1280, 1280, res=True)
conv("conv3x3 l3 1280->1280 +res", 9, 16, 1280, 1280, res=True)
tconv("tconv l0 320", 9216, 320)
tconv("tconv l2 1280", 576, 1280)
for lvl, M, C in (("l0", M0, 320), ("l1", M1, 640), ("l2", M2, 1280)):
    lin(f"linear {lvl} {C}->{C} +res", M, C, C, res=True)
    lin(f"in {lvl} {C}->{C} ln_out", M, C, C, ln_out=True)
    lin(f"out {lvl} {C}->{C} +res gn_out", M, C, C, res=True, gn_out=True)
    lin(f"qkv {lvl} {C}->{3 * C} ln", M, C, 3 * C, bias=False, ln=True)
    lin(f"geglu {lvl} {C}->{8 * C} ln", M, C, 8 * C, geglu=True, ln=True)
    lin(f"ff2 {lvl} {4 * C}->{C} +res", M, 4 * C, C, res=True)
lin("linear l3 1280->1280 +res", M3, 1280, 1280, res=True)
lin("init ff geglu 512->4096", M0, 512, 4096, geglu=True)

def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)
if args.json:
    print(json.dumps({"card": card(), "batch": args.batch, "lib": os.environ.get("VC_B200_LIB", "default"), "rows": rows}))
else:
    print(f"{card()}  batch {args.batch}")
    for r in rows:
        bw = f" {r['gbs']:7.0f} GB/s" if r["gbs"] is not None else ""
        print(f"{r['name']:32s} {r['tflops']:8.1f} TFLOP/s {r['us']:9.1f} us{bw}")
