"""FP8 tap-GEMM (gemm_tap_kernel<BN, true>, csrc/gemm_tap.cu) and the absmax kernel, through the ops wrappers.

The reference is an emulation on the SAME quantised operands: s_a = max|A| / 448 (1 if 0), q_a = e4m3(fp32(a) * (1 / s_a)) after
clamping to +-448 (torch.float8_e4m3fn rounds to nearest even), q_w / s_w from ops.pack_fp8, the tap sum of q_a * q_w in float64,
times s_a * s_w[n], then the fp16 epilogue (bias, GEGLU, residual, folded LayerNorm) in float64.  Only the kernel's summation
and the final fp16 rounding separate the two, so the bound per element is

    C8 * (K_total / 32 + 2) * 2^-13 * S  +  half an fp16 ulp of (|ref| + err)        S = sum |q_a| |q_w| s_a s_w (+ |bias| + |res|)

The e4m3 products are exact in fp32.  Hopper's fp8 wgmma adds each k32 step into the accumulator with fewer bits than fp32
(about 14 significant bits, as publicly reported for H800 / H100 fp8 GEMMs), so the unit per step is 2^-13 rather than 2^-24, summed over
the K_total / 32 steps.  That is the worst case of the summation, not of fp8 quantisation, which the emulation shares.
test prints the ratio err / bound of every case.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

C8 = 1.0
U8 = 2.0 ** -13
ERF_EPS = 1.5e-6
RATIOS = {}


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


def f16(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def quant_act(a_list):
    """(q_a fp64 per source, s_a): the kernel's activation quantisation over every source."""
    amax = max(float(a.abs().max()) for a in a_list)
    sa = torch.tensor(amax, dtype=torch.float32) / 448.0 if amax > 0 else torch.tensor(1.0)
    inv = torch.tensor(1.0, dtype=torch.float32) / sa
    qs = [(a.float() * inv.cuda()).clamp(-448, 448).to(torch.float8_e4m3fn).double() for a in a_list]
    return qs, float(sa)


def tap_ref(qa_img, qw, taps):
    """qa_img [Z, Y, X, K], qw [taps, N, K]; out[z, y, x, n] = sum_tap sum_k qa[z, y + dy, x + dx, k] qw[tap, n, k] (zero outside)."""
    Z, Y, X, K = qa_img.shape
    p = max(max(abs(dx), abs(dy)) for dx, dy in taps)
    pad = F.pad(qa_img, (0, 0, p, p, p, p))
    out = 0
    for t, (dx, dy) in enumerate(taps):
        sh = pad[:, p + dy:p + dy + Y, p + dx:p + dx + X]
        out = out + sh @ qw[t].T
    return out


def bound(S, ktot, ref, extra=0.0):
    err = C8 * (ktot / 32 + 2) * U8 * S + extra
    return err + 2.0 ** -11 * (ref.abs() + err) + 2.0 ** -24


def check(name, out, ref, bnd):
    err = (out.double() - ref).abs()
    ratio = float((err / bnd).max())
    RATIOS[name] = ratio
    print(name, "max err", float(err.max()), "ratio", ratio)
    assert torch.isfinite(out).all(), name
    assert ratio <= 1.0, (name, ratio)


def w8_of(ops, w16, taps):
    q, s = ops.pack_fp8(w16, taps)
    return ops.Fp8Weight(q, s), q.double().view(taps, -1, w16.shape[1]), s.double()


# ------------------------------------------------------------------------------------------------------------- absmax
@pytest.mark.parametrize("two", [False, True])
def test_absmax_matches_torch(ops, two):
    x = f16((1000, 320), 1, 3.0)
    x2 = f16((1000, 640), 2, 5.0) if two else None
    big = torch.zeros(1024, 1000, dtype=torch.float16, device="cuda")
    xv = big[:1000, 8:328]                       # a strided view: pitch 1000
    xv.copy_(x)
    am = ops.absmax(xv, x2)
    want = max(x.abs().max(), x2.abs().max()) if two else x.abs().max()
    assert float(am) == float(want)
    assert float(ops.absmax(torch.zeros(256, 64, dtype=torch.float16, device="cuda"))) == 0.0


# ------------------------------------------------------------------------------------------------------------- exact quantisation
@pytest.mark.parametrize("K", [32, 320])
def test_quantisation_bit_exact(ops, K):
    """One nonzero weight per output channel: every output is one e4m3 product, so the accumulation is exact and the fp16 result
    pins the kernel's activation rounding (e4m3, round to nearest even, satfinite) and scales bit for bit."""
    M, N = 300, 128
    x = f16((M, K), 30, 3.0)
    x[0, 0] = -x.abs().max() * 1.0001                      # the amax element: q = -448 exactly
    w = torch.zeros(N, K, dtype=torch.float16)
    g = torch.Generator().manual_seed(31)
    cols = torch.randint(0, K, (N,), generator=g)
    w[torch.arange(N), cols] = (torch.randn(N, generator=g) * 0.1).half()
    w = w.cuda()
    w8, qw, sw = w8_of(ops, w, 1)
    y = ops.linear(x, w8)
    (qa,), sa = quant_act([x])
    acc = (qa.float() @ qw[0].float().T)                   # one nonzero product per element: exact in fp32
    ref = (acc * (torch.tensor(sa, dtype=torch.float32) * sw.float().cpu()).cuda()).half()
    assert torch.equal(y, ref), float((y.float() - ref.float()).abs().max())


# ------------------------------------------------------------------------------------------------------------- linear
# N -> tile width the fp8 dispatcher picks: 32, 64, 96 (N=192), 128, and N=320 (64: no 160-wide fp8 tile)
@pytest.mark.parametrize("K", [320, 640, 960, 1280, 1920, 2560])
@pytest.mark.parametrize("N", [32, 64, 192, 320, 640])
def test_linear_fp8(ops, K, N):
    M = 300                                               # ragged M
    x, w = f16((M, K), 3), f16((N, K), 4, 0.05)
    bias = (torch.randn(N) * 0.1).cuda()
    res = f16((M, N), 5)
    w8, qw, sw = w8_of(ops, w, 1)
    y = ops.linear(x, w8, bias=bias, res=res)
    (qa,), sa = quant_act([x])
    acc = qa @ qw[0].T
    ref = acc * (sa * sw) + bias.double() + res.double()
    S = (qa.abs() @ qw[0].abs().T) * (sa * sw) + bias.double().abs() + res.double().abs()
    check(f"linear K{K} N{N}", y, ref, bound(S, K, ref))


def test_linear_fp8_two_sources_and_ln_part(ops):
    M, K1, K2, N = 257, 640, 320, 640
    x, x2, w = f16((M, K1), 6), f16((M, K2), 7, 4.0), f16((N, K1 + K2), 8, 0.05)
    w8, qw, sw = w8_of(ops, w, 1)
    y, st = ops.linear(x, w8, x2=x2, ln_out=True)
    (qa, qa2), sa = quant_act([x, x2])
    q = torch.cat([qa, qa2], 1)
    ref = (q @ qw[0].T) * (sa * sw)
    S = (q.abs() @ qw[0].abs().T) * (sa * sw)
    check("linear two sources", y, ref, bound(S, K1 + K2, ref))
    # the LayerNorm statistics gathered in the epilogue describe the fp16 output as stored (the fp16 kernel's contract)
    yd = y.double()
    mean, var = yd.mean(1), yd.var(1, unbiased=False)
    assert torch.allclose(st[:, 0].double(), mean, atol=1e-4, rtol=1e-4)
    assert torch.allclose(st[:, 1].double(), 1.0 / torch.sqrt(var + 1e-5), rtol=1e-3)


def test_linear_fp8_folded_layernorm(ops):
    M, K, N = 333, 640, 1920
    x = f16((M, K), 9, 2.0) + 0.5
    w, g, b = torch.randn(N, K) * 0.05, torch.rand(K) + 0.5, torch.randn(K) * 0.1
    w16, cs16, b2 = ops.fold_layernorm(w, g, b)
    w8, qw, sw = w8_of(ops, w16.cuda(), 1)
    cs = ops.fp8_colsum(w8)
    assert torch.allclose(cs.double(), (qw[0] * sw[:, None]).sum(1), rtol=1e-5, atol=1e-6)
    st = ops.layernorm_stats(x)
    y = ops.linear(x, w8, bias=b2.cuda(), ln=(st, cs))
    (qa,), sa = quant_act([x])
    mean, rstd = st[:, 0:1].double(), st[:, 1:2].double()
    acc = (qa @ qw[0].T) * (sa * sw)
    ref = rstd * (acc - mean * cs.double()) + b2.double().cuda()
    S = rstd * (qa.abs() @ qw[0].abs().T) * (sa * sw)
    extra = rstd * (mean.abs() * cs.double().abs() + acc.abs()) * 2.0 ** -22
    check("folded LN", y, ref, bound(S, K, ref, extra))


def test_linear_fp8_geglu(ops):
    M, K, N2 = 200, 640, 2 * 2560
    x = f16((M, K), 10)
    w, b = torch.randn(N2, K) * 0.05, torch.randn(N2) * 0.1
    wp, bp = ops.pack_geglu(w, b)
    w8, qw, sw = w8_of(ops, wp.cuda(), 1)
    y = ops.linear(x, w8, bias=bp.cuda(), geglu=True)
    (qa,), sa = quant_act([x])
    acc = (qa @ qw[0].T) * (sa * sw) + bp.double().cuda()
    S = (qa.abs() @ qw[0].abs().T) * (sa * sw)
    # undo the per-tile interleave: tile t holds values [t*64, t*64+64) then the matching gates
    bn, half = 128, 64
    nt = N2 // bn
    a = acc.view(M, nt, 2, half)
    val, gate = a[:, :, 0].reshape(M, -1), a[:, :, 1].reshape(M, -1)
    Sv, Sg = S.view(M, nt, 2, half)[:, :, 0].reshape(M, -1), S.view(M, nt, 2, half)[:, :, 1].reshape(M, -1)
    ref = val * F.gelu(gate)
    ev, eg = C8 * (K / 32 + 2) * U8 * Sv, C8 * (K / 32 + 2) * U8 * Sg
    extra = ev * F.gelu(gate).abs() + val.abs() * (1.13 * eg + ERF_EPS * (gate.abs() + 1))
    check("geglu", y, ref, extra + 2.0 ** -11 * (ref.abs() + extra) + 2.0 ** -24)


# ------------------------------------------------------------------------------------------------------------- convolutions
@pytest.mark.parametrize("K,N,H,W", [(320, 320, 12, 20), (640, 640, 9, 16), (960, 640, 8, 8), (1280, 1280, 5, 8)])
def test_conv3x3_fp8_gn_part(ops, K, N, H, W):
    frames = 3
    x, w = f16((frames * H * W, K), 11), f16((N, K, 3, 3), 12, 0.02)
    bias = (torch.randn(frames, N) * 0.1).cuda()
    w9 = ops.pack_conv3x3(w)
    w8, qw, sw = w8_of(ops, w9, 9)
    y = ops.conv3x3(x, frames, H, W, w8, bias=bias, bias_z_div=1, gn_out=True)
    (qa,), sa = quant_act([x])
    taps = [(t % 3 - 1, t // 3 - 1) for t in range(9)]
    img = qa.view(frames, H, W, K)
    ref = (tap_ref(img, qw, taps) * (sa * sw)).reshape(-1, N) + bias.double().repeat_interleave(H * W, 0)
    S = (tap_ref(img.abs(), qw.abs(), taps) * (sa * sw)).reshape(-1, N) + bias.double().abs().repeat_interleave(H * W, 0)
    check(f"conv3x3 K{K} N{N}", y, ref, bound(S, 9 * K, ref))
    # GroupNorm from the epilogue's partial sums against GroupNorm computed from the stored fp16 output
    g, b = torch.rand(N).cuda() + 0.5, torch.randn(N).cuda() * 0.1
    with_parts = ops.groupnorm(y, frames, g, b, 1e-5, False)
    y_plain = y.clone()                       # no _vc_gn: statistics pass
    plain = ops.groupnorm(y_plain, frames, g, b, 1e-5, False)
    assert (with_parts.float() - plain.float()).abs().max() <= 4e-3


def test_conv3x3_fp8_two_sources(ops):
    frames, H, W, K1, K2, N = 2, 8, 16, 640, 320, 320
    x, x2, w = f16((frames * H * W, K1), 13), f16((frames * H * W, K2), 14, 3.0), f16((N, K1 + K2, 3, 3), 15, 0.02)
    w8, qw, sw = w8_of(ops, ops.pack_conv3x3(w), 9)
    y = ops.conv3x3(x, frames, H, W, w8, x2=x2)
    (qa, qa2), sa = quant_act([x, x2])
    img = torch.cat([qa, qa2], 1).view(frames, H, W, K1 + K2)
    taps = [(t % 3 - 1, t // 3 - 1) for t in range(9)]
    ref = (tap_ref(img, qw, taps) * (sa * sw)).reshape(-1, N)
    S = (tap_ref(img.abs(), qw.abs(), taps) * (sa * sw)).reshape(-1, N)
    check("conv3x3 two sources", y, ref, bound(S, 9 * (K1 + K2), ref))


def test_conv_temporal_fp8_residual(ops):
    B, T, HW, C = 2, 5, 48, 640
    x, w, res = f16((B * T * HW, C), 16), f16((C, C, 3, 1, 1), 17, 0.03), f16((B * T * HW, C), 18)
    bias = (torch.randn(C) * 0.1).cuda()
    w8, qw, sw = w8_of(ops, ops.pack_conv_temporal(w), 3)
    y = ops.conv_temporal(x, B, T, HW, w8, bias=bias, res=res)
    (qa,), sa = quant_act([x])
    img = qa.view(B, 1, T * HW, C)
    taps = [((t - 1) * HW, 0) for t in range(3)]
    ref = (tap_ref(img, qw, taps) * (sa * sw)).reshape(-1, C) + bias.double() + res.double()
    S = (tap_ref(img.abs(), qw.abs(), taps) * (sa * sw)).reshape(-1, C) + bias.double().abs() + res.double().abs()
    check("temporal", y, ref, bound(S, 3 * C, ref))


def test_upconv_fp8_strided_outputs(ops):
    frames, H, W, C = 2, 6, 10, 640
    x, w = f16((frames * H * W, C), 19), f16((C, C, 3, 3), 20, 0.02)
    bias = (torch.randn(C) * 0.1).cuda()
    packs = ops.pack_upconv3x3(w)
    w8s = [w8_of(ops, p, 4) for p in packs]
    y = ops.upconv3x3(x, frames, H, W, [e[0] for e in w8s], bias=bias).view(frames, 2 * H, 2 * W, C)
    (qa,), sa = quant_act([x])
    img = qa.view(frames, H, W, C)
    for a in (0, 1):
        for b in (0, 1):
            _, qw, sw = w8s[a * 2 + b]
            taps = [((t % 2) + b - 1, (t // 2) + a - 1) for t in range(4)]
            ref = tap_ref(img, qw, taps) * (sa * sw) + bias.double()
            S = tap_ref(img.abs(), qw.abs(), taps) * (sa * sw) + bias.double().abs()
            check(f"upconv parity {a}{b}", y[:, a::2, b::2], ref, bound(S, 4 * C, ref))


# ------------------------------------------------------------------------------------------------------------- errors
def test_fp8_error_paths(ops):
    import ctypes as C
    from viewcrafter_b200 import _lib
    x, w = f16((128, 320), 21), f16((64, 320), 22)
    w8, _, _ = w8_of(ops, w, 1)
    with pytest.raises(ops.VcError, match="fp32 output"):
        ops.linear(x, w8, out_f32=True)
    am = ops.absmax(x)

    def desc(**kw):
        d = _lib.GemmDesc()
        d.a, d.lda, d.X, d.Y, d.Z, d.bx, d.by = x.data_ptr(), 320, 128, 1, 1, 128, 1
        d.K, d.K1, d.N, d.num_taps = 320, 320, 64, 1
        out = torch.empty(128, 64, dtype=torch.float16, device="cuda")
        d.out, d.ldo = out.data_ptr(), 64
        d.w, d.ldw, d.fp8, d.w_scale, d.a_amax = w8.q.data_ptr(), 320, 1, w8.scale.data_ptr(), am.data_ptr()
        for k, v in kw.items():
            setattr(d, k, v)
        return d, out

    def run(d):
        return _lib.load().vc_gemm_tap(C.byref(d), torch.cuda.current_stream().cuda_stream)

    d, out = desc()
    assert run(d) == 0
    for kw, msg in ((dict(w_scale=None), b"w_scale and a_amax"), (dict(a_amax=None), b"w_scale and a_amax"),
                    (dict(K=312, K1=312), b"K % 16")):
        d, out = desc(**kw)
        assert run(d) != 0
        assert msg in _lib.load().vc_last_error(), _lib.load().vc_last_error()
    peer = _lib.GemmPeer()
    peer.mode, peer.world = 1, 2
    d, out = desc(peer=C.cast(C.pointer(peer), C.c_void_p))
    assert run(d) != 0 and b"peer" in _lib.load().vc_last_error()


def test_report_fp8_accumulation_ratio():
    if RATIOS:
        print("fp8 err / bound: max %.3g over %d cases" % (max(RATIOS.values()), len(RATIOS)))
