"""Sweep of the tap-GEMM (gemm_tap_kernel<BN>, csrc/gemm_tap.cu + gemm_common.cuh) over its tile widths, pipeline depths, tile
counts, store paths and epilogue features, through the ops wrappers, against float64 references of the same operation.

Operands are carved out of larger NaN-filled buffers (A: rows past M and columns past K; W: columns past K and rows past
taps * N), so a load that is not clipped or zero-filled where it should be turns into NaN.  Outputs are views pre-filled with NaN
inside a buffer whose other rows and columns hold a sentinel that must come back bit-unchanged.

Tolerance, per element: the kernel rounds an fp32 value v once to the output type, so |out - ref| <= err + half an ulp of
(|ref| + err), where err bounds |v - ref|:
  * accumulation: C_ACC * (K_total + 2) * 2^-24 * (|A| @ |W|^T + |bias| + |res|), the textbook bound for a recursive fp32 sum of
    K_total products (each product of two fp16 values is exact in fp32) and the two epilogue additions.  C_ACC = 1 is that
    worst case for round-to-nearest.  The tensor cores do not document their accumulator rounding (truncation would double the
    unit roundoff), so C_ACC was chosen from a run: on an H100 80GB HBM3 the largest error over this file was 0.13 of the
    C_ACC = 1 term (errors grow like sqrt(K), the bound like K), which leaves a margin of 7x at C_ACC = 1.
    test_report_accumulation_ratio prints the ratio of every run.
  * GEGLU: the accumulation error of value and gate carried through value * gelu(gate) (|gelu'| < 1.13), plus the erf
    approximation of the epilogue (Abramowitz-Stegun 7.1.26, |err| < 1.5e-7, evaluated with rcp.approx / ex2.approx: ERF_EPS).
  * folded LayerNorm: the kernel computes rstd * (x @ W'^T - mean * colsum) from fp32 statistics and column sums; the terms are
    the rounding of that difference (the mean * colsum cancellation), the error of the fp32 column sums and the measured error
    of the fp32 statistics.
  * fused upsample-conv: its parity weights are sums of 2 or 4 taps rounded to fp16 once more (2^-11 relative).
"""
import importlib.util
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
C_ACC = 1.0
ERF_EPS = 1.5e-6
STAGES = {32: 8, 64: 7, 96: 6, 128: 5, 160: 4}         # GemmCfg<BN>::STAGES
N_OF_BN = {32: 32, 64: 64, 96: 192, 128: 128, 160: 160}
SENT = -3.0                                              # sentinel around the output views (exact in fp16 and fp32)
G = 32                                                   # guard rows above and below an output view
OUT_KINDS = ("f16", "f16_p8", "f16_p4", "f16_c4", "f32", "f32_p3")
RES_KINDS = (None, "contig", "p8", "off8", "inplace")


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


# ------------------------------------------------------------------------------------------------------------- operands
def _randn(shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def f16(shape, seed, scale=1.0):
    return _randn(shape, seed, scale).half().cuda()


def f32(shape, seed, scale=1.0):
    return _randn(shape, seed, scale).cuda()


def _nan(rows, cols, dtype=torch.float16):
    return torch.full((rows, cols), float("nan"), dtype=dtype, device="cuda")


def carve_a(vals):
    """[M, K] fp16 view with row pitch K + 24; NaN in the columns past K and in 37 rows past M."""
    M, K = vals.shape
    buf = _nan(M + 37, K + 24)
    buf[:M, :K] = vals
    return buf[:M, :K]


def carve_w(vals, pitched=True):
    """[rows, K] fp16 view with NaN in 40 rows past the end and, if pitched, in 8 columns past K (ldw = K + 8)."""
    rows, K = vals.shape
    if pitched:
        buf = _nan(rows + 40, K + 8)
        buf[:rows, :K] = vals
        return buf[:rows, :K]
    flat = torch.full(((rows + 40) * K,), float("nan"), dtype=torch.float16, device="cuda")
    v = flat[:rows * K].view(rows, K)
    v.copy_(vals)
    return v


def _pitch(n, mod, r):
    """the smallest pitch > n with pitch % mod == r (at least one guard column)"""
    return n + 1 + ((r - (n + 1)) % mod)


def out_view(M, N, kind):
    """(buffer, [M, N] view) for an output kind: f16 contiguous (TMA store when N % 32 == 0), f16 with pitch % 16 == 8 (TMA store
    without the 256-bit path), f16 with pitch % 8 == 4 (scalar), f16 contiguous but 8 bytes past a 16-byte boundary (scalar),
    f32 contiguous (256-bit when N % 8 == 0), f32 with pitch % 8 == 3 (scalar)."""
    dtype = torch.float16 if kind.startswith("f16") else torch.float32
    if kind == "f16_c4":
        buf = torch.full(((M + 2 * G) * N + 8,), SENT, dtype=dtype, device="cuda")
        v = buf[G * N + 4:G * N + 4 + M * N].view(M, N)
    else:
        pitch = {"f16": N, "f16_p8": _pitch(N, 16, 8), "f16_p4": _pitch(N, 8, 4), "f32": N, "f32_p3": _pitch(N, 8, 3)}[kind]
        buf = torch.full((M + 2 * G, pitch), SENT, dtype=dtype, device="cuda")
        v = buf[G:G + M, :N]
    v.fill_(float("nan"))
    return buf, v


def check_sentinel(buf, v, what):
    """everything of buf outside the view v still holds the sentinel, bit for bit"""
    keep = v.clone()
    v.fill_(SENT)
    ok = torch.equal(buf, torch.full_like(buf, SENT))
    v.copy_(keep)
    assert ok, f"{what}: a store landed outside the output view"


def res_view(vals, kind):
    """residual view of the fp16 values [M, N]: contiguous; pitch % 16 == 8; offset by 8 elements (16 bytes) in a pitch % 16 == 0
    buffer.  Columns around the view are NaN."""
    M, N = vals.shape
    if kind is None:
        return None
    if kind == "contig":
        return vals.clone()
    if kind == "p8":
        buf = _nan(M, _pitch(N, 16, 8))
        buf[:, :N] = vals
        return buf[:, :N]
    if kind == "off8":
        buf = _nan(M, 16 * -(-(N + 9) // 16))
        buf[:, 8:8 + N] = vals
        return buf[:, 8:8 + N]
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------------------------- tolerance
def half_ulp(x, dtype):
    """half an ulp of |x| in the output type (subnormals included)"""
    lo, man = (-14, 10) if dtype == torch.float16 else (-126, 23)
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** (lo - man - 1)))).clamp_min(lo)
    return torch.exp2(e - man - 1)


def acc_err(k_total, absacc, extra_abs=0.0):
    """bound of |v - ref| for a K_total-long fp32 dot product plus the epilogue additions (|bias| + |res| in extra_abs)"""
    return C_ACC * (k_total + 2) * U * (absacc + extra_abs)


worst = {"ratio": 0.0}                                   # largest (|out - ref| - half ulp) / (C_ACC = 1 accumulation term) seen


def bound_of(ref, err, dtype):
    return err + half_ulp(ref.abs() + err, dtype)


def check(out, ref, err, what, acc1=None):
    """out: kernel output (fp16 / fp32); ref: float64 reference; err: bound of the pre-rounding error (float64 tensor)."""
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    d = (out.double() - ref).abs()
    hu = half_ulp(ref.abs() + err, out.dtype)
    bad = ~(d <= err + hu)                               # NaN is bad
    if acc1 is not None:
        worst["ratio"] = max(worst["ratio"], float(((d - hu).clamp_min(0) / acc1.clamp_min(1e-30)).max()))
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} / {bad.numel()} elements outside the bound; first at flat index {i}: "
                             f"out {float(out.flatten()[i])} ref {float(ref.flatten()[i]):.6g} bound {float((err + hu).flatten()[i]):.3g}; "
                             f"max err {float(d.nan_to_num(float('inf')).max()):.4g}")


# ------------------------------------------------------------------------------------------------------------- linear
class Lin:
    """One linear problem [x | x2] @ w^T (+ bias) (+ res) with its float64 reference."""

    def __init__(self, M, K, N, seed, K2=0, bias=True, res=True, wscale=None):
        Kt = K + K2
        self.M, self.K, self.K2, self.N = M, K, K2, N
        self.x = carve_a(f16((M, K), seed))
        self.x2 = carve_a(f16((M, K2), seed + 1)) if K2 else None
        self.w = carve_w(f16((N, Kt), seed + 2, wscale if wscale is not None else Kt ** -0.5))
        self.b = f32((N,), seed + 3) if bias else None
        self.r = f16((M, N), seed + 4) if res else None
        a64 = self.x.double() if not K2 else torch.cat([self.x, self.x2], 1).double()
        w64 = self.w.double()
        self.a64, self.w64 = a64, w64
        self.mm = a64 @ w64.t()
        self.absacc = a64.abs() @ w64.abs().t()
        self.k_total = Kt

    def ref(self, with_res=True):
        ref = self.mm.clone()
        extra = torch.zeros_like(ref)
        if self.b is not None:
            ref += self.b.double()
            extra += self.b.double().abs()
        if with_res and self.r is not None:
            ref += self.r.double()
            extra += self.r.double().abs()
        return ref, acc_err(self.k_total, self.absacc, extra), self.k_total * U * (self.absacc + extra)

    def run(self, ops, out_kind="f16", res_kind="contig", **kw):
        """-> (output view, buffer); checks the sentinel"""
        buf, out = out_view(self.M, self.N, out_kind)
        res = None
        if res_kind == "inplace":
            out.copy_(self.r)
            res = out
        elif res_kind is not None:
            res = res_view(self.r, res_kind)
        y = ops.linear(self.x, self.w, bias=self.b, res=res, out=out, out_f32=out_kind.startswith("f32"), x2=self.x2, **kw)
        if isinstance(y, tuple):
            y = y[0]
        assert y.data_ptr() == out.data_ptr()
        check_sentinel(buf, out, f"{out_kind}/{res_kind}")
        return out

    def check(self, ops, what, out_kind="f16", res_kind="contig"):
        out = self.run(ops, out_kind, res_kind)
        ref, err, acc1 = self.ref(with_res=res_kind is not None)
        check(out, ref, err, what, acc1)
        return out


@pytest.mark.parametrize("N", [8, 32, 48, 64, 96, 192, 128, 200, 224, 512, 160, 320, 480])
def test_tile_width_and_ragged_n(ops, N):
    """Every tile width (pick_bn) with whole and ragged last n-tiles: N = 200 stores its tail on the scalar path, N = 224 takes the
    TMA store with a 96-column last tile.  K = 136: two whole k-blocks and an 8-column one."""
    case = Lin(347, 136, N, seed=N)
    for ok in ("f16", "f32"):
        case.check(ops, f"N={N} {ok}", out_kind=ok)


@pytest.mark.parametrize("BN", [32, 64, 96, 128, 160])
def test_pipeline_depth(ops, BN):
    """Per-tile iteration counts of 1, S - 1, S, S + 1 and 2 S + 1 (S = ring stages of the tile width), K below one k-block, and
    a two-source K split whose second slab is not a whole k-block.  3 m-tiles, the last one ragged."""
    S, N = STAGES[BN], N_OF_BN[BN]
    assert ops._lib.load().vc_gemm_tile_n(N, 0) == BN
    M = 128 * 3 - 37
    for K in (64, 64 * (S - 1), 64 * S, 64 * S + 8, 64 * 2 * S + 24, 8, 24, 40):
        Lin(M, K, N, seed=1000 + K).check(ops, f"BN={BN} K={K}")
    for K2 in (8, 24, 72):
        Lin(M, 64 * (S - 1), N, seed=2000 + K2, K2=K2).check(ops, f"BN={BN} K1={64 * (S - 1)} K2={K2}")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("which", ["1", "2", "3", "sms-1", "sms", "sms+1", "2sms+1"])
def test_tile_count_vs_sm_count(ops, which):
    """One n-tile, t m-tiles (the last one ragged: M = 128 t - 37) around the SM count: idle CTAs, exactly one tile per CTA, CTAs that
    run two or three tiles.  Iterations per tile below (K = 200) and above (K = 392) the ring depth of BN = 128."""
    sms = _sms()
    t = {"1": 1, "2": 2, "3": 3, "sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "2sms+1": 2 * sms + 1}[which]
    for K in (200, 392):
        Lin(128 * t - 37, K, 128, seed=3000 + t + K).check(ops, f"t={t} K={K}")


@pytest.mark.parametrize("N", [32, 48, 64, 192, 200, 224, 320])
def test_store_paths_with_residual(ops, N):
    """Every output kind x every residual layout, with and without bias.  Every store path rounds the same fp32 value once, so
    for one (A, W, bias, res) all fp16 outputs and the fp16 rounding of the fp32 outputs must be bit-identical."""
    M, K = 347, 200
    for bias in (False, True):
        case = Lin(M, K, N, seed=4000 + N + bias, bias=bias)
        for rk in RES_KINDS:
            outs = {}
            for ok in OUT_KINDS:
                if rk == "inplace" and ok.startswith("f32"):
                    continue                            # the residual is fp16: in place only into an fp16 output
                outs[ok] = case.check(ops, f"N={N} bias={bias} out={ok} res={rk}", out_kind=ok, res_kind=rk)
            base = outs["f16"]
            for ok, o in outs.items():
                o16 = o.half() if o.dtype == torch.float32 else o
                assert torch.equal(o16.view(torch.int16), base.view(torch.int16)), f"N={N} bias={bias} res={rk}: {ok} differs from f16"


# ------------------------------------------------------------------------------------------------------------- conv3x3
def _rows(t4):                                          # [n, c, h, w] -> [(n h w), c]
    n, c, h, w = t4.shape
    return t4.permute(0, 2, 3, 1).reshape(n * h * w, c)


class Conv:
    """conv3x3 (stride 1, pad 1) on channels-last rows, optionally with a K-split second source and per-z bias rows."""

    def __init__(self, frames, H, W, Ci, Co, seed, C2=0, bias_rows=1, bias_z_div=0, res=True):
        self.frames, self.H, self.W, self.Co, self.C2, self.bzd = frames, H, W, Co, C2, bias_z_div
        Ct = Ci + C2
        xi = _randn((frames, Ct, H, W), seed).half()
        wc = _randn((Co, Ct, 3, 3), seed + 1, (9 * Ct) ** -0.5).half()
        self.x = carve_a(_rows(xi[:, :Ci]).cuda())
        self.x2 = carve_a(_rows(xi[:, Ci:]).cuda()) if C2 else None
        self.w9 = carve_w(_pack_conv3x3(wc).cuda(), pitched=False)
        self.b = f32((bias_rows, Co) if bias_z_div else (Co,), seed + 2) if bias_rows else None
        self.M = frames * H * W
        self.r = f16((self.M, Co), seed + 3) if res else None
        x64, w64 = xi.double().cuda(), wc.double().cuda()
        self.mm = _rows(F.conv2d(x64, w64, padding=1))
        self.absacc = _rows(F.conv2d(x64.abs(), w64.abs(), padding=1))
        self.k_total = 9 * Ct

    def bias_rows64(self, shift=0):
        if self.b is None:
            return None
        if not self.bzd:
            return self.b.double().expand(self.M, self.Co)
        z = (torch.arange(self.frames, device="cuda") // self.bzd + shift) % self.b.shape[0]
        return self.b.double()[z].repeat_interleave(self.H * self.W, 0)

    def ref(self, with_res=True, bias_shift=0):
        ref, extra = self.mm.clone(), torch.zeros_like(self.mm)
        b = self.bias_rows64(bias_shift)
        if b is not None:
            ref += b
            extra += b.abs()
        if with_res and self.r is not None:
            ref += self.r.double()
            extra += self.r.double().abs()
        return ref, acc_err(self.k_total, self.absacc, extra), self.k_total * U * (self.absacc + extra)

    def check(self, ops, what, out_kind="f16", res_kind="contig"):
        buf, out = out_view(self.M, self.Co, out_kind)
        res = None
        if res_kind == "inplace":
            out.copy_(self.r)
            res = out
        elif res_kind is not None:
            res = res_view(self.r, res_kind)
        y = ops.conv3x3(self.x, self.frames, self.H, self.W, self.w9, bias=self.b, res=res, x2=self.x2, bias_z_div=self.bzd,
                        out_f32=out_kind.startswith("f32"), out=out)
        assert y.data_ptr() == out.data_ptr()
        check_sentinel(buf, out, what)
        ref, err, acc1 = self.ref(with_res=res_kind is not None)
        check(out, ref, err, what, acc1)
        return out


def _pack_conv3x3(w):
    from viewcrafter_b200 import ops
    return ops.pack_conv3x3(w)


def test_conv3x3_store_paths_per_z_bias_and_residual(ops):
    """Per-z bias rows (bias_z_div = 2 over 4 frames) with every output kind x residual layout; bit-identical across store paths."""
    case = Conv(4, 5, 12, 72, 64, seed=5000, bias_rows=2, bias_z_div=2)
    for rk in RES_KINDS:
        outs = {}
        for ok in OUT_KINDS:
            if rk == "inplace" and ok.startswith("f32"):
                continue
            outs[ok] = case.check(ops, f"conv out={ok} res={rk}", out_kind=ok, res_kind=rk)
        for ok, o in outs.items():
            o16 = o.half() if o.dtype == torch.float32 else o
            assert torch.equal(o16.view(torch.int16), outs["f16"].view(torch.int16)), f"conv res={rk}: {ok} differs from f16"


# (frames, H, W, Ci, Co): multi-row boxes (W divides 128, bx = W, by = 128 / W; W < 32 makes TMA-store boxes narrower than 32 rows),
# one 128-pixel box per row segment (other W), H = 1 / 3 / not a multiple of by, 1-3 frames, Ci = 8 / 72
CONV_GEOMS = [(1, 3, 1, 8, 32), (2, 1, 2, 72, 32), (3, 70, 4, 8, 96), (1, 20, 8, 72, 32), (2, 3, 16, 8, 64), (3, 5, 32, 72, 32),
              (1, 3, 64, 8, 96), (2, 2, 128, 72, 32), (3, 1, 5, 8, 32), (1, 3, 7, 72, 64), (2, 11, 12, 8, 32), (1, 3, 96, 72, 32),
              (2, 3, 200, 8, 96), (1, 9, 1, 72, 64), (2, 33, 2, 8, 32)]


@pytest.mark.parametrize("frames,H,W,Ci,Co", CONV_GEOMS)
def test_conv3x3_geometry(ops, frames, H, W, Ci, Co):
    case = Conv(frames, H, W, Ci, Co, seed=6000 + H * 7 + W, bias_rows=frames, bias_z_div=1)
    case.check(ops, f"conv {frames}x{H}x{W} Ci={Ci} Co={Co}")


def test_conv3x3_concat_k2_8(ops):
    """Channel concat whose second source is 8 channels (K1 = 64, K2 = 8: one k-block of the first map, a ragged one of the second)."""
    for H, W in ((5, 16), (3, 7)):
        Conv(2, H, W, 64, 32, seed=6500 + W, C2=8).check(ops, f"concat {H}x{W}")


# ------------------------------------------------------------------------------------------------------------- temporal / upsample conv
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [1, 2, 3, 25])
def test_conv_temporal(ops, B, T):
    C, N = 72, 64
    for HW in (1, 7, 130):
        x5 = _randn((B, C, T, HW, 1), 7000 + T + HW).half()
        w = _randn((N, C, 3, 1, 1), 7001, (3 * C) ** -0.5).half()
        b, r = f32((N,), 7002), f16((B * T * HW, N), 7003)
        rows = lambda t5: t5.permute(0, 2, 3, 4, 1).reshape(B * T * HW, -1)
        x64, w64 = x5.double().cuda(), w.double().cuda()
        ref = rows(F.conv3d(x64, w64, padding=(1, 0, 0))) + b.double() + r.double()
        absacc = rows(F.conv3d(x64.abs(), w64.abs(), padding=(1, 0, 0)))
        extra = b.double().abs() + r.double().abs()
        out = ops.conv_temporal(carve_a(rows(x5).cuda()), B, T, HW, carve_w(ops.pack_conv_temporal(w).cuda(), pitched=False), bias=b, res=r)
        check(out, ref, acc_err(3 * C, absacc, extra), f"temporal B={B} T={T} HW={HW}", 3 * C * U * (absacc + extra))


@pytest.mark.parametrize("Co", [32, 96, 160])
def test_upconv3x3(ops, Co):
    frames, H, Ci = 2, 3, 40
    for W in (1, 2, 7, 16):
        x = _randn((frames, Ci, H, W), 8000 + W).half()
        w = _randn((Co, Ci, 3, 3), 8001, (9 * Ci) ** -0.5).half()
        b = f32((Co,), 8002)
        packs = [carve_w(p.cuda(), pitched=False) for p in ops.pack_upconv3x3(w.float())]
        y = ops.upconv3x3(carve_a(_rows(x).cuda()), frames, H, W, packs, bias=b)
        xu = F.interpolate(x.double().cuda(), scale_factor=2, mode="nearest")
        w64 = w.double().cuda()
        ref = _rows(F.conv2d(xu, w64, padding=1)) + b.double()
        absacc = _rows(F.conv2d(xu.abs(), w64.abs(), padding=1))
        err = acc_err(4 * Ci, absacc, b.double().abs()) + 2.0 ** -11 * absacc      # + the fp16 rounding of the summed parity taps
        check(y, ref, err, f"upconv W={W} Co={Co}")


# ------------------------------------------------------------------------------------------------------------- epilogue features
def _ln_problem(M, C, N, seed, geglu=False):
    """x (row means != 0), LayerNorm gamma / beta and a projection, folded (fold_layernorm / pack_geglu_ln)."""
    x = carve_a((_randn((M, C), seed, 1.5) + 0.7).half().cuda())
    g, be = f32((C,), seed + 1) + 1.0, f32((C,), seed + 2, 0.3)
    w, bias = f32((N, C), seed + 3, C ** -0.5), f32((N,), seed + 4, 0.2)
    return x, g, be, w, bias


def _ln_ref(ops, x, w16, cs, b2):
    """float64 reference of LayerNorm (no affine: gamma is folded into w16) -> linear, and the bound of the folded evaluation."""
    x64, w64 = x.double(), w16.double()
    mean = x64.mean(1, keepdim=True)
    var = x64.var(1, unbiased=False, keepdim=True)
    rstd = torch.rsqrt(var + 1e-5)
    st = ops.layernorm_stats(x.contiguous())
    dm = (st[:, :1].double() - mean).abs()
    dr = (st[:, 1:].double() / rstd - 1).abs()
    # the statistics themselves are not what this file tests, but their error must be small for the bound to mean anything
    assert float(dm.max()) < 1e-5 and float(dr.max()) < 1e-5, (float(dm.max()), float(dr.max()))
    pre = F.layer_norm(x64, (x.shape[1],), eps=1e-5) @ w64.t()
    acc, absacc = x64 @ w64.t(), x64.abs() @ w64.abs().t()
    cs64 = w64.sum(1)
    csf = cs.double()
    K = x.shape[1]
    e = (C_ACC * (K + 2) * U * absacc                      # x @ W'^T in fp32
         + 2 * U * (acc.abs() + (mean * csf).abs())        # acc - mean * colsum: the cancellation, rounded in fp32
         + mean.abs() * (csf - cs64).abs()                 # fp32 column sums
         + dm * csf.abs()) * rstd * (1 + dr) + dr * pre.abs() + 2 * U * pre.abs()
    return st, pre + b2.double(), e, b2.double().abs()


@pytest.mark.parametrize("out_kind", ["f16", "f16_p8", "f16_p4"])
@pytest.mark.parametrize("ln", [False, True])
def test_geglu(ops, out_kind, ln):
    """GEGLU on the accumulator fragments (BN = 128), with and without a folded LayerNorm, on the TMA and scalar output paths."""
    M, C, N2 = 347, 200, 256
    if ln:
        x, g, be, w, bias = _ln_problem(M, C, N2, seed=9000)
        wp, bp, cs = ops.pack_geglu_ln(w, bias, g, be)
        w16, cs_unpacked, b2 = ops.fold_layernorm(w, g, be, bias)
        st, h, eh, babs = _ln_ref(ops, x, w16, cs_unpacked, b2)
        eh = eh + C_ACC * 2 * U * babs
        kw = dict(ln=(st, cs))
    else:
        x = carve_a(f16((M, C), 9100))
        w16, bias = f16((N2, C), 9101, C ** -0.5), f32((N2,), 9102, 0.5)
        wp, bp = ops.pack_geglu(w16, bias)
        x64, w64 = x.double(), w16.double()
        h = x64 @ w64.t() + bias.double()
        eh = acc_err(C, x64.abs() @ w64.abs().t(), bias.double().abs())
        kw = {}
    val, gate, ev, eg = h[:, :N2 // 2], h[:, N2 // 2:], eh[:, :N2 // 2], eh[:, N2 // 2:]
    gelu = 0.5 * gate * (1 + torch.erf(gate / math.sqrt(2)))
    ref = val * gelu
    err = ev * gelu.abs() + (val.abs() + ev) * (1.13 * eg + 0.5 * gate.abs() * ERF_EPS) + 4 * U * ref.abs()
    buf, out = out_view(M, N2 // 2, out_kind)
    y = ops.linear(x, carve_w(wp), bias=bp, geglu=True, out=out, **kw)
    assert y.data_ptr() == out.data_ptr()
    check_sentinel(buf, out, "geglu")
    check(out, ref, err, f"geglu ln={ln} out={out_kind}")


@pytest.mark.parametrize("out_kind", ["f16", "f16_p4", "f32_p3"])
def test_folded_layernorm_with_residual(ops, out_kind):
    M, C, N = 347, 200, 320
    x, g, be, w, bias = _ln_problem(M, C, N, seed=9200)
    w16, cs, b2 = ops.fold_layernorm(w, g, be, bias)
    st, ref, err, babs = _ln_ref(ops, x, w16, cs, b2)
    r = f16((M, N), 9205)
    ref, err = ref + r.double(), err + C_ACC * 2 * U * (babs + r.double().abs() + ref.abs())
    buf, out = out_view(M, N, out_kind)
    ops.linear(x, carve_w(w16), bias=b2, res=res_view(r, "p8"), out=out, out_f32=out_kind.startswith("f32"), ln=(st, cs))
    check_sentinel(buf, out, "folded LN")
    check(out, ref, err, f"folded LN out={out_kind}")


@pytest.mark.parametrize("out_kind", ["f16", "f16_c4"])
@pytest.mark.parametrize("res_kind", RES_KINDS)
def test_ln_out_with_residual_views(ops, res_kind, out_kind):
    """ln_out (contiguous outputs: TMA store, and scalar store from a pointer 8 bytes off): the output is bit-identical to the call
    without it, and the statistics describe the stored output."""
    case = Lin(347, 136, 320, seed=9300)
    buf, out = out_view(case.M, case.N, out_kind)
    res = None if res_kind is None else (out.copy_(case.r) if res_kind == "inplace" else res_view(case.r, res_kind))
    y, st = ops.linear(case.x, case.w, bias=case.b, res=res, out=out, ln_out=True)
    check_sentinel(buf, out, "ln_out")
    ref, err, acc1 = case.ref(with_res=res_kind is not None)
    check(y, ref, err, f"ln_out out={out_kind} res={res_kind}", acc1)
    y0 = case.run(ops, out_kind, res_kind)
    assert torch.equal(y.view(torch.int16), y0.view(torch.int16))
    yc = y.clone()                                          # 16-byte aligned copy: the statistics kernel reads 8-channel vectors
    yf = yc.double()
    mean, rstd = yf.mean(1), torch.rsqrt(yf.var(1, unbiased=False) + 1e-5)
    assert float((st[:, 0] - mean).abs().max()) < 2e-4 * max(1.0, float(mean.abs().max()))
    assert float(((st[:, 1] - rstd) / rstd).abs().max()) < 2e-4
    assert float((st - ops.layernorm_stats(yc)).abs().max()) < 1e-3


def _gn_compare(ops, y, samples, what):
    """GroupNorm from the producer's records vs GroupNorm of a record-free clone (statistics pass): equal up to fp32 summation order.
    Both read 16-byte aligned copies of y (the GroupNorm kernels read 8-channel vectors); the first one carries y's records."""
    assert ops.gn_part_of(y) is not None
    C = y.shape[1]
    g, b = f32((C,), 9400), f32((C,), 9401)
    n0 = ops.gn_from_parts_calls
    ya = y.clone()
    ya._vc_gn = ops.gn_part_of(y)
    a = ops.groupnorm(ya, samples, g, b, 1e-5, False)
    assert ops.gn_from_parts_calls - n0 == 1, "expected the partial-sum path"
    c = ops.groupnorm(y.clone(), samples, g, b, 1e-5, False)
    d = (a.double() - c.double()).abs()
    tol = 2 * half_ulp(c.double().abs(), torch.float16) + 1e-4
    assert bool((d <= tol).all()), f"{what}: GroupNorm from the records differs from the stored output's by up to {float(d.max()):.4g}"


def _force_gn_parts(ops, monkeypatch):
    monkeypatch.setattr(ops, "GN_FROM_PRODUCER", 2)
    monkeypatch.setattr(ops, "GN_PARTS_MIN_MB", 0.0)
    monkeypatch.setattr(ops, "REPRODUCIBLE", False)


@pytest.mark.parametrize("out_kind", ["f16", "f16_c4"])
@pytest.mark.parametrize("res_kind", RES_KINDS)
def test_gn_out_with_residual_views(ops, monkeypatch, res_kind, out_kind):
    """gn_out (linear and conv3x3, contiguous outputs on the TMA and the scalar store path): the output is bit-identical to the
    call without it, and the GroupNorm records describe the stored output (residual included)."""
    _force_gn_parts(ops, monkeypatch)
    case = Lin(347, 136, 320, seed=9500)
    y = case.run(ops, out_kind, res_kind, gn_out=True)
    check(y, *case.ref(with_res=res_kind is not None)[:2], f"gn_out linear out={out_kind} res={res_kind}")
    assert torch.equal(y.view(torch.int16), case.run(ops, out_kind, res_kind).view(torch.int16))
    _gn_compare(ops, y, 1, f"linear out={out_kind} res={res_kind}")
    conv = Conv(2, 5, 16, 64, 320, seed=9600)
    buf, out = out_view(conv.M, conv.Co, out_kind)
    res = None if res_kind is None else (out.copy_(conv.r) if res_kind == "inplace" else res_view(conv.r, res_kind))
    yc = ops.conv3x3(conv.x, conv.frames, conv.H, conv.W, conv.w9, bias=conv.b, res=res, out=out, gn_out=True)
    check_sentinel(buf, out, "gn_out conv")
    check(yc, *conv.ref(with_res=res_kind is not None)[:2], f"gn_out conv out={out_kind} res={res_kind}")
    _gn_compare(ops, yc, conv.frames, f"conv out={out_kind} res={res_kind}")


# ------------------------------------------------------------------------------------------------------------- negative controls
def _outside(pert, ref, bound):
    return bool(((pert - ref).abs() > bound).any())


def test_tolerance_rejects_plausible_kernel_bugs(ops):
    """Reference side only: each perturbed reference a kernel bug would produce falls outside the bound somewhere."""
    S = STAGES[128]
    case = Lin(347, 64 * S + 8, 128, seed=9700)
    ref, err, _ = case.ref()
    bound = bound_of(ref, err, torch.float16)
    assert _outside(ref - case.r.double(), ref, bound), "residual omitted"
    kl = 64 * S                                               # the last k-block holds columns [64 S, 64 S + 8)
    no_last = case.a64[:, :kl] @ case.w64[:, :kl].t() + case.b.double() + case.r.double()
    assert _outside(no_last, ref, bound), "last k-block omitted"
    shifted = torch.cat([ref[:, 1:], ref[:, -1:]], 1)
    assert _outside(shifted, ref, bound), "output columns shifted by one"
    conv = Conv(4, 5, 12, 72, 64, seed=9800, bias_rows=2, bias_z_div=2)
    cref, cerr, _ = conv.ref()
    wrong_z, _, _ = conv.ref(bias_shift=1)
    assert _outside(wrong_z, cref, bound_of(cref, cerr, torch.float16)), "bias of the wrong z row"


# ------------------------------------------------------------------------------------------------------------- grid size
def _grid_tool():
    spec = importlib.util.spec_from_file_location("gemm_grid_check", os.path.join(ROOT, "tools", "gemm_grid_check.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_results_do_not_depend_on_the_grid_size(ops, monkeypatch, tmp_path):
    """tools/gemm_grid_check.py runs a fixed set of GEMMs in child processes whose grids are cut to 1, 3 and 8 CTAs (VC_SM_COUNT,
    read once per process); outputs, GroupNorm records and LayerNorm statistics must equal this process's full-grid results."""
    _force_gn_parts(ops, monkeypatch)
    tool = _grid_tool()
    full = tool.run_all(ops)
    procs = {}
    for k in (1, 3, 8):
        env = dict(os.environ, VC_SM_COUNT=str(k))
        env.pop("VC_REPRODUCIBLE", None)
        procs[k] = subprocess.Popen([sys.executable, os.path.join(ROOT, "tools", "gemm_grid_check.py"), str(tmp_path / f"grid{k}.pt")],
                                    stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
    for k, p in procs.items():
        out, _ = p.communicate(timeout=400)
        print(out[-3000:])
        assert p.returncode == 0 and "GEMM_GRID_CHECK_OK" in out, f"VC_SM_COUNT={k}"
        got = torch.load(tmp_path / f"grid{k}.pt")
        assert sorted(got) == sorted(full)
        for name, d in full.items():
            for key, t in d.items():
                assert torch.equal(got[name][key], t), f"VC_SM_COUNT={k}: {name} {key} differs from the full grid"


def test_report_accumulation_ratio(ops):
    """Largest observed (|out - ref| - half ulp) / (K_total * 2^-24 * |A| @ |W|^T) of this run (printed; the bound uses C_ACC)."""
    print(f"GEMM_SWEEP worst accumulation ratio {worst['ratio']:.4g} (C_ACC = {C_ACC})")
    assert worst["ratio"] <= C_ACC
