"""Micro-benchmark of the attention kernels at the U-Net shapes (development tool)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from viewcrafter_b200 import ops
def t(fn, reps=5):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3
T = 25
for name, HW, heads in (("l0", 9216, 5), ("l1", 2304, 10), ("l2", 576, 20), ("l3", 144, 20)):
    C = heads * 64
    qkv = (torch.randn(T * HW, 3 * C, device="cuda") * 0.7).half()
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    dt = t(lambda: ops.flash_attn(q, k, v, T, HW, HW, heads))
    fl = 4.0 * T * heads * HW * HW * 64
    # accuracy vs fp32 reference on one (frame, head)
    qq, kk, vv = (x[:HW, :64].float() for x in (q, k, v))
    ref = torch.softmax(qq @ kk.t() * 0.125, -1) @ vv
    out = ops.flash_attn(q, k, v, T, HW, HW, heads)[:HW, :64].float()
    err = (out - ref).abs()
    print(f"self-attn {name} N={HW:5d} heads={heads:2d}: {dt*1e3:7.3f} ms {fl/dt/1e12:7.1f} TFLOP/s   max err {float(err.max()):.2e} mean {float(err.mean()):.2e} (ref absmax {float(ref.abs().max()):.2f})")
    dt2 = t(lambda: ops.temporal_attn(q, k, v, T, HW, heads))
    by = 4.0 * T * HW * C * 2
    print(f"temporal  {name} sites={HW:5d}: {dt2*1e6:8.1f} us  {by/dt2/1e9:7.1f} GB/s")
kv = (torch.randn(333, 2 * 320, device="cuda") * 0.7).half()
q = (torch.randn(T * 9216, 320, device="cuda") * 0.7).half()
for Nk in (77, 256):
    dt = t(lambda: ops.flash_attn(q, kv[:Nk, :320], kv[:Nk, 320:], T, 9216, Nk, 5, kv_shared=True))
    print(f"cross-attn l0 Nk={Nk:3d}: {dt*1e6:8.1f} us")
