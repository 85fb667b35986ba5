"""The small kernels of csrc/misc.cu and the GEGLU epilogue's GELU against high-precision references, at their edges.

  * erf-GELU: ops.gelu_f16 on all 65,536 fp16 bit patterns and the GEGLU epilogue (ops.linear(geglu=True) with value weights 0, value
    bias 1 and identity gate weights, so the output is fp16(gelu(x)) of every finite fp16 x) within the bound of tests/gelu_ref.py;
    inf / NaN inputs give the class torch's F.gelu gives;
  * timestep_embedding: every t in 0..999 and fps values, at dims 320, 321 (the zero pad column) and 64, against the float64 sinusoid
    within a derived bound; small_linear against float64 within a recursive-summation bound, SiLU inputs near +-90 included;
  * layout, cast and resampling kernels: bit-exact against torch, with NaN-filled outputs and sentinel columns around the written ones,
    at sizes past one grid-stride round (sm_count * 16 blocks of 256 threads);
  * the wrappers' argument checks, on views carved inside larger allocations (a missing check shows up as a missing exception).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import gelu_ref as G

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
U32 = 2.0 ** -24
SENTINEL = -1234.5


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


def _grid_round(ops):
    """Elements one grid-stride round of the 256-thread, sm_count * 16-block kernels covers."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256


def _dirty(nbytes):
    """Leave a freed block of all-ones bytes (NaN as fp16 and fp32) in the caching allocator, so that an output the kernel allocates
    next with this size starts out NaN instead of stale data that might happen to be right."""
    torch.full((nbytes,), 255, dtype=torch.uint8, device="cuda")


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _same(got, ref):
    """Bit-identical, except that any NaN may stand for any NaN."""
    ref = ref.to(got.device)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(_bits(got)[~nan], _bits(ref)[~nan])


# ---------------------------------------------------------------------------------------------- erf-GELU
def test_gelu_on_every_fp16_bit_pattern(ops):
    allx = torch.arange(1 << 16, dtype=torch.int32).to(torch.int16).view(torch.float16)
    fin = torch.isfinite(allx)
    out = ops.gelu_f16(allx.cuda()).cpu()
    x = allx[fin].numpy()
    r, at = G.worst_ratio(out[fin].numpy(), x)
    # the GEGLU epilogue: columns 0..63 of the packed weight are values (0 x + 1), 64..127 the gates (x itself)
    w = torch.cat([torch.zeros(64, 64), torch.eye(64)]).cuda()
    b = torch.cat([torch.ones(64), torch.zeros(64)]).cuda()
    wp, bp = ops.pack_geglu(w, b)
    xf = allx[fin].reshape(992, 64)
    geglu = ops.linear(xf.cuda(), wp, bias=bp, geglu=True).cpu().reshape(-1)
    rg, atg = G.worst_ratio(geglu.numpy(), x)
    differ = int((_bits(geglu) != _bits(out[fin])).sum())
    print(f"gelu_f16: worst error / bound {r:.4f} at x={at:.5g}; GEGLU epilogue: {rg:.4f} at x={atg:.5g}; "
          f"the two paths differ in {differ} of {x.size} outputs")
    ref16 = G.gelu_ref(x).astype(np.float16).astype(np.float64)
    for name, o in (("gelu_f16", out[fin].numpy()), ("GEGLU epilogue", geglu.numpy())):
        ulps = np.abs(o.astype(np.float64) - ref16) / (2 * G.half_ulp_fp16(np.abs(ref16)))
        worst = np.argsort(-ulps)[:3]
        print(f"{name}: at most {ulps.max():.0f} fp16 ulps from the rounded exact GELU, at x = {[float(x[k]) for k in worst]}")
    assert r <= 1.0 and rg <= 1.0
    ref = F.gelu(allx[~fin].float().cuda()).cpu()
    got = out[~fin].float()
    print(f"non-finite inputs: {allx[~fin].unique().numel()} patterns; kernel +inf -> {float(got[allx[~fin] == math.inf][0])}")
    for cls in (torch.isnan, torch.isposinf, torch.isneginf, lambda t: t == 0):
        assert torch.equal(cls(got), cls(ref))


# ---------------------------------------------------------------------------------------------- embeddings
def _embedding_bound(t, dim):
    """|kernel - float64 sinusoid| per element.  freq = expf(fl(fl(-ln 1e4) j) / half): the constant, the product and the quotient
    round once each, so the exponent a = ln(1e4) j / half is within 3u relative and exp moves by 3u a; expf is within 2 ulp (4u);
    arg = fl(t freq) rounds once more.  So |arg - t freq| <= t freq (3 a + 5) u, and cos / sin move by at most that, plus their own
    2 ulp (4u, and one u of absolute slack for results near 0)."""
    half = dim // 2
    j = torch.arange(half, dtype=torch.float64)
    a = math.log(10000.0) * j / half
    freq = torch.exp(-a)
    arg_err = t.double()[:, None] * freq[None] * (3 * a + 5)[None] * U32
    ref_arg = t.double()[:, None] * freq[None]
    cos, sin = torch.cos(ref_arg), torch.sin(ref_arg)
    ref = torch.cat([cos, sin] + ([torch.zeros(t.shape[0], 1, dtype=torch.float64)] if dim % 2 else []), 1)
    bound = torch.cat([arg_err + 4 * U32 * cos.abs() + U32, arg_err + 4 * U32 * sin.abs() + U32]
                      + ([torch.zeros(t.shape[0], 1, dtype=torch.float64)] if dim % 2 else []), 1)
    return ref, bound


@pytest.mark.parametrize("dim", [320, 321, 64])
def test_timestep_embedding_every_step_and_fps(ops, dim):
    from oracle import lvdm_oracle as O
    t = torch.cat([torch.arange(1000), torch.tensor([1, 3, 10, 24, 30, 60])])
    e = ops.timestep_embedding(t.cuda(), dim).cpu().double()
    ref, bound = _embedding_bound(t, dim)
    zero_pad = (bound == 0)
    assert torch.equal(e[zero_pad], ref[zero_pad])
    ratio = ((e - ref).abs() / bound.clamp_min(1e-300))[~zero_pad]
    oracle = ((O.timestep_embedding(t, dim).double() - ref).abs() / bound.clamp_min(1e-300))[~zero_pad]
    print(f"dim={dim}: kernel worst error / bound {float(ratio.max()):.3g} (max |err| {float((e - ref).abs().max()):.3g}); "
          f"the reference's fp32 formula {float(oracle.max()):.3g}")
    assert float(ratio.max()) <= 1.0 and float(oracle.max()) <= 1.0


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("bias,add", [(False, False), (True, False), (True, True), (False, True)])
@pytest.mark.parametrize("K", [320, 1280, 333])
def test_small_linear_against_float64(ops, K, bias, add, silu):
    """Each lane sums ceil(K / 32) products in order (fma), five shuffle levels add the lanes, then bias and add: at most
    m = ceil(K / 32) + 7 roundings on any path, |err| <= gamma_m (sum |x_k w_k| + |b| + |add|).  SiLU = x / (1 + expf(-x)): expf
    within 2 ulp, the sum and the quotient round once, so silu(x) is within 6u relative; where expf(-x) overflows (x < -88.7) the
    kernel returns -0 and |silu(x)| < 2^-100 is the error.  Inputs include x near +-90."""
    N = 1280
    g = torch.Generator().manual_seed(K + 2 * bias + add)
    w = torch.randn(N, K, generator=g) * 0.05
    b = torch.randn(N, generator=g) if bias else None
    worst = 0.0
    for rows in range(1, 7):
        x = torch.randn(rows, K, generator=g) * 3.0
        x[:, :8] = torch.tensor([88.5, -88.5, 89.0, -89.0, 90.0, -90.0, 91.5, -91.5])
        a = torch.randn(rows, N, generator=g) if add else None
        out = ops.small_linear(x.cuda(), w.cuda(), None if b is None else b.cuda(), silu_in=silu,
                               add=None if a is None else a.cuda()).cpu().double()
        xd = x.double()
        xs = xd * torch.sigmoid(xd) if silu else xd
        ref = xs @ w.double().T
        mag = xs.abs() @ w.double().abs().T
        if silu:
            mag_silu = (6 * U32 * xs.abs() + 2.0 ** -100) @ w.double().abs().T
        if b is not None:
            ref, mag = ref + b.double(), mag + b.double().abs()
        if a is not None:
            ref, mag = ref + a.double(), mag + a.double().abs()
        m = -(-K // 32) + 7
        bound = m * U32 / (1 - m * U32) * mag + (mag_silu if silu else 0.0)
        r = float(((out - ref).abs() / bound).max())
        assert torch.isfinite(out).all() and r <= 1.0, (rows, r)
        worst = max(worst, r)
    print(f"small_linear K={K} bias={bias} add={add} silu={silu}: worst error / bound {worst:.3g} over rows 1..6")


# ---------------------------------------------------------------------------------------------- layout / cast / resampling
def _edge_f32(n, seed):
    """n fp32 values: every fp32 -> fp16 rounding edge (overflow, the 65520 tie, round-half-even ties, subnormals and their ties, -0,
    +-inf, NaN), then random bit patterns (every class, all exponents), then N(0, 1)."""
    edges = [65504.0, 65519.99, 65520.0, 65536.0, 1e10, -65520.0, math.inf, -math.inf, math.nan, -0.0, 0.0,
             2.0 ** -24, 2.0 ** -25, -2.0 ** -25, 2.0 ** -25 * (1 + 2 ** -20), 3 * 2.0 ** -25, 5 * 2.0 ** -25, 2.0 ** -14 - 2.0 ** -25,
             1e-45, -1e-40, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(1 + 2.0 ** -11), 2048 + 1.0, 2048 + 3.0, 6.1e-5, 1.0 / 3.0]
    g = torch.Generator().manual_seed(seed)
    k = (n - len(edges)) // 2
    rnd_bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (k,), generator=g, dtype=torch.int64).to(torch.int32).view(torch.float32)
    return torch.cat([torch.tensor(edges, dtype=torch.float32), rnd_bits, torch.randn(n - len(edges) - k, generator=g)])


def test_cast_f16_rounding_edges(ops):
    n = 2 * _grid_round(ops) + 77
    x = _edge_f32(n, 1)
    _dirty(2 * n)
    _same(ops.cast_f16(x.cuda()), x.half())


@pytest.mark.parametrize("shape,c_off,pitch", [((2, 4, 5, 96, 160), 4, 8), ((1, 4, 1, 576, 1024), 0, 8), ((1, 3, 1, 5, 9), 2, 13),
                                               ((2, 4, 3, 40, 64), 0, 4)])
def test_ncthw_to_rows_writes_only_its_columns(ops, shape, c_off, pitch):
    B, C, T, H, W = shape
    rows = B * T * H * W
    x = _edge_f32(B * C * T * H * W, 2).reshape(shape)
    buf = torch.full((rows + 6, pitch + 3), SENTINEL, dtype=torch.float16, device="cuda")
    out = buf[3:rows + 3, 1:pitch + 1]                                   # pitch + 3 columns apart, inside the sentinel frame
    out[:, c_off:c_off + C] = math.nan
    ops.ncthw_to_rows(x.cuda(), out, c_off)
    want = torch.full(buf.shape, SENTINEL, dtype=torch.float16)          # built on its own: every cell but the block is the sentinel
    want[3:rows + 3, 1 + c_off:1 + c_off + C] = x.permute(0, 2, 3, 4, 1).reshape(rows, C).half()
    _same(buf, want)


@pytest.mark.parametrize("shape,pitch", [((2, 4, 5, 96, 160), 8), ((1, 3, 1, 5, 9), 13)])
def test_rows_to_ncthw_and_rows_f16_to_nchw_read_only_their_columns(ops, shape, pitch):
    B, C, T, H, W = shape
    rows = B * T * H * W
    g = torch.Generator().manual_seed(3)
    big = torch.full((rows + 2, pitch + 2), math.nan)
    big[1:rows + 1, 1:C + 1] = torch.randn(rows, C, generator=g) * 100
    big32 = big.cuda()
    _dirty(4 * B * C * T * H * W)
    got = ops.rows_to_ncthw(big32[1:rows + 1, 1:pitch + 1], B, C, T, H, W)
    _same(got, big[1:rows + 1, 1:C + 1].reshape(B, T, H, W, C).permute(0, 4, 1, 2, 3))
    big16 = big.half()
    _dirty(4 * B * C * T * H * W)
    got = ops.rows_f16_to_nchw(big16.cuda()[1:rows + 1, 1:pitch + 1], B * T, C, H, W)
    _same(got, big16[1:rows + 1, 1:C + 1].float().reshape(B * T, H, W, C).permute(0, 3, 1, 2))


def test_add_f16(ops):
    n = 2 * _grid_round(ops) + 66
    a, b = _edge_f32(n, 4).half(), _edge_f32(n, 5).flip(0).half()
    _dirty(2 * n)
    _same(ops.add_f16(a.cuda(), b.cuda()), (a.float() + b.float()).half())


def _nchw(rows, N, H, W):
    return rows.reshape(N, H, W, -1).permute(0, 3, 1, 2)


def _rows(nchw):
    return nchw.permute(0, 2, 3, 1).reshape(-1, nchw.shape[1]).contiguous()


@pytest.mark.parametrize("N,H,W,C", [(2, 36, 64, 320), (3, 5, 7, 64), (1, 9, 1, 8)])     # 737,280 16-byte vectors: > 1 round
def test_upsample2x_against_interpolate(ops, N, H, W, C):
    g = torch.Generator().manual_seed(N * H * W + C)
    x = (torch.randn(N * H * W, C, generator=g) * 10).half().cuda()
    _dirty(2 * 4 * x.numel())
    got = ops.upsample2x(x, N, H, W)
    _same(got, _rows(F.interpolate(_nchw(x, N, H, W), scale_factor=2, mode="nearest")))


@pytest.mark.parametrize("N,H,W,C,pad", [(1, 576, 1024, 128, (0, 1)), (2, 36, 64, 320, (1, 1)), (3, 9, 13, 64, (1, 1)),
                                         (2, 7, 11, 8, (0, 1)), (1, 1, 1, 16, (1, 1))])
def test_im2col_s2_against_unfold(ops, N, H, W, C, pad):
    g = torch.Generator().manual_seed(H * W + C)
    x = (torch.randn(N * H * W, C, generator=g) * 10).half().cuda()
    Ho, Wo = (H + sum(pad) - 3) // 2 + 1, (W + sum(pad) - 3) // 2 + 1
    _dirty(2 * N * Ho * Wo * 9 * C)
    got, ho, wo = ops.im2col_s2(x, N, H, W, pad_lo=pad[0], pad_hi=pad[1])
    assert (ho, wo) == (Ho, Wo)
    cols = F.unfold(F.pad(_nchw(x, N, H, W), (pad[0], pad[1], pad[0], pad[1])), 3, stride=2)        # [N, C * 9, L], (c, tap)
    ref = cols.reshape(N, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(N * Ho * Wo, 9 * C)                # tap-major rows
    _same(got, ref)
    del cols, ref, got


# ---------------------------------------------------------------------------------------------- wrapper argument checks
def test_wrappers_reject_views_the_kernels_cannot_take(ops):
    """Every view lies inside a larger 16-byte aligned allocation, so that a missing check could only give a wrong result."""
    VcError = ops.VcError
    N, H, W, C = 2, 4, 6, 16
    rows = N * H * W
    big = torch.randn(rows + 8, 2 * C, device="cuda").half()
    dense = big[:rows].reshape(-1)[:rows * C].view(rows, C)              # contiguous, aligned
    for f in (lambda v, n: ops.upsample2x(v, n, H, W), lambda v, n: ops.im2col_s2(v, n, H, W)):
        f(dense, N)
        with pytest.raises(VcError):
            f(big[:rows, :C], N)                                         # column view: pitch 2C, not C
        with pytest.raises(VcError):
            f(big[:rows - 1].reshape(-1)[:(rows - 1) * C].view(rows - 1, C), N)   # one row short of N H W
        with pytest.raises(VcError):
            f(big[:rows], N - 1)                                         # more rows than N H W
    a = big.reshape(-1)[:64]
    ops.add_f16(a, big.reshape(-1)[64:128])
    with pytest.raises(VcError):
        ops.add_f16(a, big.reshape(-1)[64:126])                          # shapes differ
    with pytest.raises(VcError):
        ops.add_f16(big[:4, :C], big[4:8, :C])                           # not contiguous
    with pytest.raises(VcError):
        ops.add_f16(a[:63], a[:63])                                      # odd count
    x5 = torch.randn(N, 4, 1, H, W, device="cuda")
    out = torch.zeros(rows + 4, 8, device="cuda", dtype=torch.float16)
    ops.ncthw_to_rows(x5, out[:rows], 4)
    for bad, c_off in ((out[:rows].float(), 0), (out[:rows, ::2], 0), (out[:rows], 5), (out[:rows, :6], 4), (out[:rows - 1], 0),
                       (out[:rows + 1], 0), (out[1:rows + 1, 1:], -1)):              # c_off = -1 would still land inside out
        with pytest.raises(VcError):
            ops.ncthw_to_rows(x5, bad, c_off)
    r32 = torch.randn(rows + 4, 8, device="cuda")
    ops.rows_to_ncthw(r32[:rows, :4], N, 4, 1, H, W)
    h16 = torch.randn(2 * rows, 8, device="cuda").half()                  # read as fp32 it would still lie inside this allocation
    for bad in (r32[:rows - 1], r32[:rows + 1], r32[:rows, ::2], r32[:rows, :3], h16[:rows]):
        with pytest.raises(VcError):
            ops.rows_to_ncthw(bad, N, 4, 1, H, W)
    r16 = r32.half()
    ops.rows_f16_to_nchw(r16[:rows, 2:6], N, 4, H, W)
    for bad in (r16[:rows - 1], r16[:rows + 1], r16[:rows, ::2], r16[:rows, :3]):
        with pytest.raises(VcError):
            ops.rows_f16_to_nchw(bad, N, 4, H, W)
