"""Micro-benchmark of the GroupNorm-statistics-from-the-producer path (ops.GN_FROM_PRODUCER): cost of gn_out in the producing GEMMs and
time of the consuming GroupNorm with / without the producer's partial sums, at the headline shapes (25 frames, 72x128 latents).
Device ms by CUDA events, 5 reps after warm-up.      python tools/gn_parts_micro.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from viewcrafter_b200 import ops

ops.GN_FROM_PRODUCER = 2
ops.GN_PARTS_MIN_MB = 0.0


def t(fn, reps=5):
    fn(); fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3


T = 25
torch.manual_seed(0)
for name, H, W, C in (("l0", 72, 128, 320), ("l1", 36, 64, 640), ("l2", 18, 32, 1280)):
    M = T * H * W
    x = (torch.randn(M, C, device="cuda") * 0.8).half()
    r = (torch.randn(M, C, device="cuda") * 0.8).half()
    w9 = (torch.randn(9 * C, C, device="cuda") * (1.0 / (3 * C ** 0.5))).half()
    w3 = (torch.randn(3 * C, C, device="cuda") * (1.0 / (1.7 * C ** 0.5))).half()
    w1 = (torch.randn(C, C, device="cuda") * (1.0 / C ** 0.5)).half()
    g, b = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.1
    prods = (("conv3x3+res", lambda go: ops.conv3x3(x, T, H, W, w9, res=r, gn_out=go)),
             ("tconv", lambda go: ops.conv_temporal(x, 1, T, H * W, w3, gn_out=go)),
             ("linear+res", lambda go: ops.linear(x, w1, res=r, gn_out=go)))
    for pn, f in prods:
        t0, t1 = t(lambda: f(False)), t(lambda: f(True))
        print(f"[gn-parts] {name} C={C:4d} producer {pn:12s}: plain {t0*1e6:8.1f} us   with gn_out {t1*1e6:8.1f} us   ({(t1/t0-1)*100:+.1f} %)")
    y = ops.conv3x3(x, T, H, W, w9, res=r, gn_out=True)
    yc = y.clone()                                     # no partial sums attached -> statistics-pass kernel
    for cn, samples in (("4-D", T), ("5-D", 1)):
        ta, tb = t(lambda: ops.groupnorm(yc, samples, g, b, 1e-5, True)), t(lambda: ops.groupnorm(y, samples, g, b, 1e-5, True))
        err = float((ops.groupnorm(yc, samples, g, b, 1e-5, True).float() - ops.groupnorm(y, samples, g, b, 1e-5, True).float()).abs().max())
        by = 2.0 * M * C * 2
        print(f"[gn-parts] {name} C={C:4d} groupnorm {cn}: statistics pass {ta*1e6:8.1f} us ({by/ta/1e9:6.0f} GB/s)   from producer sums {tb*1e6:8.1f} us "
              f"({by/tb/1e9:6.0f} GB/s r+w once)   |diff| {err:.2e}")
# B = 2 (what a CFG step runs): per-frame GroupNorm over 50 frames at every level -- the tensor sizes ops.GN_PARTS_MIN_MB chooses between
for name, H, W, C in (("l0", 72, 128, 320), ("l1", 36, 64, 640), ("l2", 18, 32, 1280), ("l3", 9, 16, 1280)):
    M = 2 * T * H * W
    x = (torch.randn(M, C, device="cuda") * 0.8).half()
    w9 = (torch.randn(9 * C, C, device="cuda") * (1.0 / (3 * C ** 0.5))).half()
    g, b = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.1
    y = ops.conv3x3(x, 2 * T, H, W, w9, gn_out=True)
    yc = y.clone()
    for cn, samples in (("4-D B=2", 2 * T), ("5-D B=2", 2)):
        ta, tb = t(lambda: ops.groupnorm(yc, samples, g, b, 1e-5, True)), t(lambda: ops.groupnorm(y, samples, g, b, 1e-5, True))
        by = 2.0 * M * C * 2
        print(f"[gn-parts] {name} C={C:4d} {M * C * 2 / 1e6:6.0f} MB groupnorm {cn}: statistics pass {ta*1e6:8.1f} us   from producer sums {tb*1e6:8.1f} us")
