"""Micro-benchmark of the tap-GEMM on the shapes that dominate a 25x72x128 U-Net forward (development tool)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from viewcrafter_b200 import ops

dev = "cuda"
def t(fn, reps=20):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3

def rnd(*s): return (torch.randn(*s, device=dev) * 0.05).half()
T = 25
rows = []
def lin(name, M, K, N, res=False, geglu=False, bias=True):
    x, w = rnd(M, K), rnd(N, K)
    b = torch.zeros(N, device=dev) if bias else None
    if geglu: w, b = ops.pack_geglu(w, b)
    r = rnd(M, N) if res else None
    dt = t(lambda: ops.linear(x, w, bias=b, res=r, geglu=geglu))
    rows.append((name, 2.0 * M * K * N / dt / 1e12, dt * 1e6))
def conv(name, H, W, Ci, Co, res=False):
    x, w9 = rnd(T * H * W, Ci), rnd(9 * Co, Ci)
    b = torch.zeros(Co, device=dev); r = rnd(T * H * W, Co) if res else None
    dt = t(lambda: ops.conv3x3(x, T, H, W, w9, bias=b, res=r))
    rows.append((name, 2.0 * T * H * W * 9 * Ci * Co / dt / 1e12, dt * 1e6))
def tconv(name, HW, C):
    x, w3 = rnd(T * HW, C), rnd(3 * C, C)
    b = torch.zeros(C, device=dev)
    dt = t(lambda: ops.conv_temporal(x, 1, T, HW, w3, bias=b))
    rows.append((name, 2.0 * T * HW * 3 * C * C / dt / 1e12, dt * 1e6))

M0, M1, M2, M3 = T * 9216, T * 2304, T * 576, T * 144
conv("conv3x3 l0 320->320", 72, 128, 320, 320, res=True)
conv("conv3x3 l0 960->320", 72, 128, 960, 320)
conv("conv3x3 l1 640->640", 36, 64, 640, 640, res=True)
conv("conv3x3 l2 1280->1280", 18, 32, 1280, 1280, res=True)
conv("conv3x3 l3 1280->1280", 9, 16, 1280, 1280, res=True)
tconv("tconv l0 320", 9216, 320)
tconv("tconv l2 1280", 576, 1280)
lin("linear l0 320->320 +res", M0, 320, 320, res=True)
lin("qkv l0 320->960", M0, 320, 960, bias=False)
lin("geglu l0 320->2560", M0, 320, 2560, geglu=True)
lin("ff2 l0 1280->320 +res", M0, 1280, 320, res=True)
lin("linear l1 640->640 +res", M1, 640, 640, res=True)
lin("qkv l1 640->1920", M1, 640, 1920, bias=False)
lin("geglu l1 640->5120", M1, 640, 5120, geglu=True)
lin("ff2 l1 2560->640 +res", M1, 2560, 640, res=True)
lin("qkv l2 1280->3840", M2, 1280, 3840, bias=False)
lin("geglu l2 1280->10240", M2, 1280, 10240, geglu=True)
lin("ff2 l2 5120->1280 +res", M2, 5120, 1280, res=True)
lin("linear l3 1280->1280", M3, 1280, 1280, res=True)
lin("init ff geglu 512->4096", M0, 512, 4096, geglu=True)
print("epilogue mode:", os.environ.get("VC_GEMM_EPI", "direct"))
for n, tf, us in rows:
    print(f"{n:28s} {tf:8.1f} TFLOP/s {us:9.1f} us")
