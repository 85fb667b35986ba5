"""Op-level parity of the sm_90a kernels (called through the C ABI) against plain PyTorch fp32 references.

Tolerances: inputs/outputs are fp16 with fp32 accumulation, so the bound is a few fp16 ulps of the output
magnitude: |err| <= atol + rtol*|ref| with rtol 4e-3 (fp16 eps = 9.8e-4) unless stated.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


def rnd(*shape, seed=0, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def close(out, ref, atol, rtol=4e-3, what=""):
    out, ref = out.float(), ref.float()
    err = (out - ref).abs()
    bound = atol + rtol * ref.abs()
    bad = (err > bound)
    assert not bool(bad.any()), f"{what}: max err {float(err.max()):.4g} (ref absmax {float(ref.abs().max()):.4g}), {int(bad.sum())} / {bad.numel()} outside tolerance"


# ---------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,K,N", [(300, 320, 320), (128, 64, 512), (1000, 1280, 1280), (257, 1024, 640), (77, 1024, 320),
                                   (4096, 512, 4096), (130, 320, 64), (513, 2560, 1280)])
def test_linear(ops, M, K, N):
    x, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    b = rnd(N, seed=3, dtype=torch.float32)
    r = rnd(M, N, seed=4)
    ref = x.float() @ w.float().t()
    close(ops.linear(x, w), ref, 2e-3, what="plain")
    close(ops.linear(x, w, bias=b, res=r), ref + b + r.float(), 4e-3, what="bias+res")
    o32 = ops.linear(x, w, bias=b, out_f32=True)
    assert o32.dtype == torch.float32
    close(o32, ref + b, 1e-3, rtol=1e-3, what="f32 out")


def test_linear_inplace_residual_and_views(ops):
    M, C = 640, 320
    x = rnd(M, 3 * C, seed=5)
    w = rnd(C, C, seed=6, scale=C ** -0.5)
    h = rnd(M, C, seed=7)
    ref = x[:, C:2 * C].float() @ w.float().t() + h.float()
    ops.linear(x[:, C:2 * C], w, res=h, out=h)          # strided A view, in-place residual
    close(h, ref, 4e-3, what="inplace")


def test_linear_two_sources(ops):
    M, K1, K2, N = 384, 640, 320, 320
    a, b = rnd(M, K1, seed=8), rnd(M, K2, seed=9)
    w = rnd(N, K1 + K2, seed=10, scale=(K1 + K2) ** -0.5)
    ref = torch.cat([a, b], 1).float() @ w.float().t()
    close(ops.linear(a, w, x2=b), ref, 2e-3, what="concat-K")


@pytest.mark.parametrize("C", [320, 512, 1280])
def test_geglu(ops, C):
    M = 300
    x = rnd(M, C, seed=11)
    w = rnd(8 * C, C, seed=12, scale=C ** -0.5)
    b = rnd(8 * C, seed=13, dtype=torch.float32, scale=0.1)
    h = x.float() @ w.float().t() + b
    val, gate = h.chunk(2, dim=-1)
    ref = val * F.gelu(gate)
    wp, bp = ops.pack_geglu(w, b)
    close(ops.linear(x, wp, bias=bp, geglu=True), ref, 4e-3, what="geglu")


def test_linear_ragged_n(ops):
    M, K, N = 200, 320, 4
    x, w = rnd(M, K, seed=14), rnd(N, K, seed=15, scale=K ** -0.5)
    b = rnd(N, seed=16, dtype=torch.float32)
    out = ops.linear(x, w, bias=b, out_f32=True)
    close(out, x.float() @ w.float().t() + b, 1e-3, what="N=4")


# ---------------------------------------------------------------------------------------------- convs
def _nhwc_rows(x_nchw):
    n, c, h, w = x_nchw.shape
    return x_nchw.permute(0, 2, 3, 1).reshape(n * h * w, c).contiguous()


@pytest.mark.parametrize("frames,H,W,Ci,Co", [(2, 9, 16, 64, 128), (3, 18, 32, 320, 320), (1, 8, 128, 128, 64), (2, 5, 8, 64, 64),
                                             (1, 6, 256, 64, 32), (2, 36, 64, 320, 640), (1, 8, 16, 8, 320), (2, 8, 16, 320, 4)])
def test_conv3x3(ops, frames, H, W, Ci, Co):
    x = rnd(frames, Ci, H, W, seed=20)
    w = rnd(Co, Ci, 3, 3, seed=21, scale=(9 * Ci) ** -0.5)
    b = rnd(Co, seed=22, dtype=torch.float32)
    ref = _nhwc_rows(F.conv2d(x.float(), w.float(), b, padding=1))
    out = ops.conv3x3(_nhwc_rows(x), frames, H, W, ops.pack_conv3x3(w), bias=b, out_f32=(Co < 8))
    close(out, ref, 3e-3, what="conv3x3")


def test_conv3x3_concat_bias_per_batch_residual(ops):
    frames, H, W, C1, C2, Co = 4, 9, 16, 128, 64, 128
    a, s = rnd(frames, C1, H, W, seed=23), rnd(frames, C2, H, W, seed=24)
    w = rnd(Co, C1 + C2, 3, 3, seed=25, scale=(9 * (C1 + C2)) ** -0.5)
    b = rnd(2, Co, seed=26, dtype=torch.float32)           # one bias row per batch of 2 frames
    r = rnd(frames * H * W, Co, seed=27)
    ref = F.conv2d(torch.cat([a, s], 1).float(), w.float(), None, padding=1) + b.repeat_interleave(2, 0)[:, :, None, None]
    ref = _nhwc_rows(ref) + r.float()
    out = ops.conv3x3(_nhwc_rows(a), frames, H, W, ops.pack_conv3x3(w), bias=b, bias_z_div=2, res=r, x2=_nhwc_rows(s))
    close(out, ref, 4e-3, what="conv concat")


@pytest.mark.parametrize("B,T,HW,C", [(1, 5, 144, 320), (2, 4, 64, 128), (1, 25, 40, 64), (1, 1, 256, 64)])
def test_conv_temporal(ops, B, T, HW, C):
    x5 = rnd(B, C, T, HW, 1, seed=30)
    w = rnd(C, C, 3, 1, 1, seed=31, scale=(3 * C) ** -0.5)
    b = rnd(C, seed=32, dtype=torch.float32)
    ref5 = F.conv3d(x5.float(), w.float(), b, padding=(1, 0, 0))
    rows = lambda t5: t5.permute(0, 2, 3, 4, 1).reshape(B * T * HW, C).contiguous()
    r = rnd(B * T * HW, C, seed=33)
    out = ops.conv_temporal(rows(x5), B, T, HW, ops.pack_conv_temporal(w), bias=b, res=r)
    close(out, rows(ref5) + r.float(), 4e-3, what="conv_temporal")


def test_downsample_conv_via_im2col(ops):
    N, H, W, C = 3, 18, 32, 64
    x = rnd(N, C, H, W, seed=34)
    w = rnd(C, C, 3, 3, seed=35, scale=(9 * C) ** -0.5)
    b = rnd(C, seed=36, dtype=torch.float32)
    ref = _nhwc_rows(F.conv2d(x.float(), w.float(), b, stride=2, padding=1))
    cols, Ho, Wo = ops.im2col_s2(_nhwc_rows(x), N, H, W)
    wk = w.permute(0, 2, 3, 1).reshape(C, 9 * C).to(torch.float16).contiguous()
    out = ops.linear(cols, wk, bias=b)
    assert (Ho, Wo) == (9, 16)
    close(out, ref, 3e-3, what="stride-2 conv")


def test_upsample2x(ops):
    N, H, W, C = 2, 5, 7, 64
    x = rnd(N, C, H, W, seed=37)
    ref = _nhwc_rows(F.interpolate(x.float(), scale_factor=2, mode="nearest"))
    assert torch.equal(ops.upsample2x(_nhwc_rows(x), N, H, W).float(), ref)


# ---------------------------------------------------------------------------------------------- attention
def _attn_ref(q, k, v, heads, scale):
    B, Nq, _ = q.shape
    f = lambda t: t.float().reshape(t.shape[0], t.shape[1], heads, 64).permute(0, 2, 1, 3)
    s = torch.einsum("bhid,bhjd->bhij", f(q), f(k)) * scale
    o = torch.einsum("bhij,bhjd->bhid", s.softmax(-1), f(v))
    return o.permute(0, 2, 1, 3).reshape(B, Nq, heads * 64)


@pytest.mark.parametrize("B,heads,N", [(2, 5, 576), (1, 2, 128), (3, 1, 144), (1, 5, 2304), (2, 10, 1000)])
def test_flash_self_attention(ops, B, heads, N):
    C = heads * 64
    qkv = rnd(B * N, 3 * C, seed=40)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    ref = _attn_ref(q.reshape(B, N, C), k.reshape(B, N, C), v.reshape(B, N, C), heads, 0.125)
    out = ops.flash_attn(q, k, v, B, N, N, heads)
    close(out.reshape(B, N, C), ref, 2e-3, rtol=1e-2, what="self-attn")


@pytest.mark.parametrize("Nk", [77, 256, 16, 333])
def test_flash_cross_attention_shared_kv_and_accumulate(ops, Nk):
    B, heads, Nq = 3, 5, 200
    C = heads * 64
    q = rnd(B * Nq, C, seed=41)
    kv = rnd(Nk, 2 * C, seed=42)
    k, v = kv[:, :C], kv[:, C:]
    ref = _attn_ref(q.reshape(B, Nq, C), k.reshape(1, Nk, C).expand(B, Nk, C), v.reshape(1, Nk, C).expand(B, Nk, C), heads, 0.125)
    out = ops.flash_attn(q, k, v, B, Nq, Nk, heads, kv_shared=True)
    close(out.reshape(B, Nq, C), ref, 2e-3, rtol=1e-2, what="cross-attn")
    out2 = ops.flash_attn(q, k, v, B, Nq, Nk, heads, kv_shared=True, out=out.clone(), accumulate=True)
    close(out2.reshape(B, Nq, C), 2 * ref, 4e-3, rtol=1e-2, what="cross-attn accumulate")


def test_flash_cross_attention_per_batch_kv(ops):
    B, heads, Nq, Nk = 4, 2, 130, 93
    C = heads * 64
    q, k, v = rnd(B * Nq, C, seed=43), rnd(B * Nk, C, seed=44), rnd(B * Nk, C, seed=45)
    ref = _attn_ref(q.reshape(B, Nq, C), k.reshape(B, Nk, C), v.reshape(B, Nk, C), heads, 0.125)
    close(ops.flash_attn(q, k, v, B, Nq, Nk, heads).reshape(B, Nq, C), ref, 2e-3, rtol=1e-2, what="per-batch kv")


@pytest.mark.parametrize("T,sites,heads", [(25, 144, 5), (16, 100, 8), (1, 7, 1), (32, 33, 2)])
def test_temporal_attention(ops, T, sites, heads):
    C = heads * 64
    qkv = rnd(T * sites, 3 * C, seed=46)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    tok = lambda t: t.reshape(T, sites, C).permute(1, 0, 2)       # (site, t, c)
    ref = _attn_ref(tok(q), tok(k), tok(v), heads, 0.125).permute(1, 0, 2).reshape(T * sites, C)
    close(ops.temporal_attn(q, k, v, T, sites, heads), ref, 2e-3, rtol=5e-3, what="temporal attn")


# ---------------------------------------------------------------------------------------------- norms
@pytest.mark.parametrize("samples,rows,C,eps,silu", [(5, 144, 320, 1e-5, True), (1, 5 * 144, 640, 1e-5, True), (2, 1000, 128, 1e-6, False),
                                                    (3, 64, 2560, 1e-5, True), (25, 64, 64, 1e-6, False)])
def test_groupnorm(ops, samples, rows, C, eps, silu):
    x = rnd(samples * rows, C, seed=50, scale=2.0) + 0.5
    g, b = rnd(C, seed=51, dtype=torch.float32), rnd(C, seed=52, dtype=torch.float32)
    xr = x.float().reshape(samples, rows, C).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, g, b, eps)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(samples * rows, C)
    close(ops.groupnorm(x, samples, g, b, eps, silu), ref, 3e-3, what="groupnorm")


def test_groupnorm_concat(ops):
    samples, rows, C1, C2 = 3, 200, 640, 320
    a, s = rnd(samples * rows, C1, seed=53), rnd(samples * rows, C2, seed=54, scale=3.0)
    C = C1 + C2
    g, b = rnd(C, seed=55, dtype=torch.float32), rnd(C, seed=56, dtype=torch.float32)
    xr = torch.cat([a, s], 1).float().reshape(samples, rows, C).permute(0, 2, 1)
    ref = F.silu(F.group_norm(xr, 32, g, b, 1e-5)).permute(0, 2, 1).reshape(samples * rows, C)
    close(ops.groupnorm(a, samples, g, b, 1e-5, True, x2=s), ref, 3e-3, what="groupnorm concat")


@pytest.mark.parametrize("rows,C", [(1000, 320), (77, 512), (300, 1280), (9, 640), (5, 64)])
def test_layernorm(ops, rows, C):
    x = rnd(rows, C, seed=57, scale=2.0) + 1.0
    g, b = rnd(C, seed=58, dtype=torch.float32), rnd(C, seed=59, dtype=torch.float32)
    close(ops.layernorm(x, g, b), F.layer_norm(x.float(), (C,), g, b, 1e-5), 3e-3, what="layernorm")


@pytest.mark.parametrize("rows,C", [(300, 320), (1000, 1280)])
def test_layernorm_stats(ops, rows, C):
    x = rnd(rows, C, seed=157, scale=2.0) + 1.0
    st = ops.layernorm_stats(x)
    xf = x.float()
    close(st[:, 0], xf.mean(1), 1e-5, what="ln mean")
    close(st[:, 1], torch.rsqrt(xf.var(1, unbiased=False) + 1e-5), 1e-5, what="ln rstd")


@pytest.mark.parametrize("M,C,N", [(300, 320, 960), (9216, 320, 320), (700, 640, 1920), (1000, 1280, 3840)])
def test_linear_folded_layernorm(ops, M, C, N):
    """LayerNorm folded into the consumer GEMM (raw rows in, epilogue applies mean / rstd) vs LayerNorm -> Linear in fp32."""
    x = rnd(M, C, seed=158, scale=1.5) + 0.7                  # non-zero row means: the mean * colsum term matters
    g, b = rnd(C, seed=159, dtype=torch.float32) + 1.0, rnd(C, seed=160, dtype=torch.float32, scale=0.3)
    w = rnd(N, C, seed=161, dtype=torch.float32, scale=C ** -0.5)
    bias = rnd(N, seed=162, dtype=torch.float32, scale=0.2)
    ref = F.layer_norm(x.float(), (C,), g, b, 1e-5) @ w.t() + bias
    w16, cs, b2 = ops.fold_layernorm(w, g, b, bias)
    out = ops.linear(x, w16, bias=b2, ln=(ops.layernorm_stats(x), cs))
    close(out, ref, 6e-3, what="folded LN linear")


@pytest.mark.parametrize("M,C", [(300, 320), (2304, 640)])
def test_geglu_folded_layernorm(ops, M, C):
    x = rnd(M, C, seed=163, scale=1.5) - 0.4
    g, b = rnd(C, seed=164, dtype=torch.float32) + 1.0, rnd(C, seed=165, dtype=torch.float32, scale=0.3)
    w = rnd(8 * C, C, seed=166, dtype=torch.float32, scale=C ** -0.5)
    bias = rnd(8 * C, seed=167, dtype=torch.float32, scale=0.1)
    h = F.layer_norm(x.float(), (C,), g, b, 1e-5) @ w.t() + bias
    val, gate = h.chunk(2, dim=-1)
    wp, bp, cs = ops.pack_geglu_ln(w, bias, g, b)
    out = ops.linear(x, wp, bias=bp, geglu=True, ln=(ops.layernorm_stats(x), cs))
    close(out, val * F.gelu(gate), 8e-3, what="folded LN geglu")


# ---------------------------------------------------------------------------------------------- boundary / embedding / ddim
def test_layout_roundtrip(ops):
    B, C, T, H, W = 2, 4, 3, 5, 8
    x = rnd(B, C, T, H, W, seed=60, dtype=torch.float32)
    rows = torch.zeros(B * T * H * W, 8, device="cuda", dtype=torch.float16)
    ops.ncthw_to_rows(x, rows, 0)
    ops.ncthw_to_rows(x * 2, rows, 4)
    ref = x.permute(0, 2, 3, 4, 1).reshape(-1, C)
    assert torch.equal(rows[:, :4].float(), ref.half().float()) and torch.equal(rows[:, 4:].float(), (2 * ref).half().float())
    back = ops.rows_to_ncthw(ref.contiguous(), B, C, T, H, W)
    assert torch.equal(back, x)
    img = ops.rows_f16_to_nchw(rows, B * T, 8, H, W)
    assert torch.equal(img, rows.float().reshape(B * T, H, W, 8).permute(0, 3, 1, 2))


def test_embedding_mlp(ops):
    t = torch.tensor([999, 19], device="cuda", dtype=torch.int64)
    e = ops.timestep_embedding(t, 320)
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / half)
    args = t.cpu()[:, None].float() * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
    assert float((e.cpu() - ref).abs().max()) < 2e-4          # fp32 exp/sincos at |arg| <= 999
    w, b = rnd(1280, 320, seed=61, dtype=torch.float32, scale=0.05), rnd(1280, seed=62, dtype=torch.float32)
    add = rnd(2, 1280, seed=63, dtype=torch.float32)
    out = ops.small_linear(e, w, b, silu_in=True, add=add)
    close(out, F.linear(F.silu(e), w, b) + add, 1e-4, rtol=1e-4, what="small_linear")


@pytest.mark.parametrize("cfg,gr", [(7.5, 0.7), (7.5, 0.0), (1.0, 0.0)])
def test_ddim_update_matches_oracle(ops, cfg, gr):
    from oracle import lvdm_oracle as O
    sched = O.model_schedule(base_scale=0.3)
    tab = O.ddim_tables(sched, 50, "uniform_trailing", 1.0)
    shape = (1, 4, 5, 8, 16)
    g = torch.Generator().manual_seed(64)
    x, vc_, vu, nz = (torch.randn(shape, generator=g) for _ in range(4))
    for index in (49, 20, 0):
        step = int(tab["timesteps"][index])
        sc = O.step_scalars(tab, index)
        sa, s1 = sched["sqrt_alphas_cumprod"][step].item(), sched["sqrt_one_minus_alphas_cumprod"][step].item()
        ref_prev, ref_x0 = O.ddim_update(x, vc_, vu if cfg != 1.0 else None, sc, sa, s1, nz, cfg, gr)
        d = dict(cfg_scale=cfg, guidance_rescale=gr, sqrt_ac_t=sa, sqrt_1mac_t=s1, a_prev=float(sc[1]), sigma_t=float(sc[2]),
                 scale_t=float(sc[4]), prev_scale_t=float(sc[5]))
        xp, x0 = ops.ddim_update(x.cuda(), vc_.cuda(), vu.cuda(), nz.cuda(), d)
        close(xp.cpu(), ref_prev, 2e-5, rtol=2e-5, what=f"x_prev index {index}")
        close(x0.cpu(), ref_x0, 2e-5, rtol=2e-5, what=f"pred_x0 index {index}")


@pytest.mark.parametrize("gr", [0.0, 0.7])
def test_ddim_update_three_way_cfg_matches_oracle(ops, gr):
    """vc_ddim_update3: u + cfg_img (v_img - u) + s (v_cond - v_img) (ddim_multiplecond.py:227-233) + the shared tail."""
    from oracle import lvdm_oracle as O
    sched = O.model_schedule(base_scale=0.3)
    tab = O.ddim_tables(sched, 50, "uniform_trailing", 1.0, fixed_prev_scale=False)
    shape = (1, 4, 5, 8, 16)
    g = torch.Generator().manual_seed(65)
    x, vc_, vu, vi, nz = (torch.randn(shape, generator=g) for _ in range(5))
    for index in (49, 0):
        step = int(tab["timesteps"][index])
        sc = O.step_scalars(tab, index)
        sa, s1 = sched["sqrt_alphas_cumprod"][step].item(), sched["sqrt_one_minus_alphas_cumprod"][step].item()
        ref_prev, ref_x0 = O.ddim_update(x, vc_, vu, sc, sa, s1, nz, 7.5, gr, v_uncond_img=vi, cfg_img=2.5)
        d = dict(cfg_scale=7.5, guidance_rescale=gr, sqrt_ac_t=sa, sqrt_1mac_t=s1, a_prev=float(sc[1]), sigma_t=float(sc[2]),
                 scale_t=float(sc[4]), prev_scale_t=float(sc[5]))
        xp, x0 = ops.ddim_update(x.cuda(), vc_.cuda(), vu.cuda(), nz.cuda(), d, v_uncond_img=vi.cuda(), cfg_img=2.5)
        close(xp.cpu(), ref_prev, 5e-5, rtol=2e-5, what=f"3-way x_prev index {index}")
        close(x0.cpu(), ref_x0, 5e-5, rtol=2e-5, what=f"3-way pred_x0 index {index}")


def test_gelu_matches_torch(ops):
    x = rnd(257, 4096, seed=66, scale=2.0)
    close(ops.gelu_f16(x), torch.nn.functional.gelu(x.float()), 2e-3, rtol=2e-3, what="gelu")


def test_linear_strided_weight_view(ops):
    """w may be a column slice of a wider matrix (the VAE attention uses K = fused-QK[:, C:] as the 'weight')."""
    M, C = 300, 512
    qk = rnd(M, 2 * C, seed=70)
    ref = qk[:, :C].float() @ qk[:, C:].float().t()
    out = ops.linear(qk[:, :C], qk[:, C:], out_f32=True)
    close(out, ref, 2e-2, rtol=2e-3, what="strided w")


def test_gemm_many_tile_rounds(ops):
    """Large shapes (more tiles than SMs, several persistent rounds): odd m-tile counts, ragged M, bias + residual, GEGLU, K-split concat, 3x3 conv taps and temporal taps."""
    M = 128 * 301 + 37
    x, w = rnd(M, 320, seed=80), rnd(320, 320, seed=81, scale=320 ** -0.5)
    b, r = rnd(320, seed=82, dtype=torch.float32), rnd(M, 320, seed=83)
    close(ops.linear(x, w, bias=b, res=r), x.float() @ w.float().t() + b + r.float(), 4e-3, what="many-tile linear N=320")
    w2 = rnd(1024, 320, seed=84, scale=320 ** -0.5)
    close(ops.linear(x, w2), x.float() @ w2.float().t(), 2e-3, what="many-tile linear N=1024")
    wg = rnd(2560, 320, seed=85, scale=320 ** -0.5)
    bg = rnd(2560, seed=86, dtype=torch.float32, scale=0.1)
    hh = x.float() @ wg.float().t() + bg
    wp, bp = ops.pack_geglu(wg, bg)
    close(ops.linear(x, wp, bias=bp, geglu=True), hh[:, :1280] * F.gelu(hh[:, 1280:]), 4e-3, what="many-tile geglu")
    a2 = rnd(M, 128, seed=87)
    w3 = rnd(384, 448, seed=88, scale=448 ** -0.5)
    close(ops.linear(x, w3, x2=a2), torch.cat([x, a2], 1).float() @ w3.float().t(), 2e-3, what="many-tile concat-K")
    frames, H, W, Ci, Co = 5, 72, 128, 64, 256
    xi = rnd(frames, Ci, H, W, seed=89)
    wc = rnd(Co, Ci, 3, 3, seed=90, scale=(9 * Ci) ** -0.5)
    bc = rnd(Co, seed=91, dtype=torch.float32)
    ref = _nhwc_rows(F.conv2d(xi.float(), wc.float(), bc, padding=1))
    close(ops.conv3x3(_nhwc_rows(xi), frames, H, W, ops.pack_conv3x3(wc), bias=bc), ref, 3e-3, what="many-tile conv3x3")
    frames, H, W, Ci, Co = 41, 18, 32, 64, 128                     # 5 tiles per frame (last one ragged), odd tile count
    xi = rnd(frames, Ci, H, W, seed=92)
    wc = rnd(Co, Ci, 3, 3, seed=93, scale=(9 * Ci) ** -0.5)
    ref = _nhwc_rows(F.conv2d(xi.float(), wc.float(), None, padding=1))
    close(ops.conv3x3(_nhwc_rows(xi), frames, H, W, ops.pack_conv3x3(wc)), ref, 3e-3, what="many-tile conv3x3 ragged")
    B, T, HW, C = 1, 5, 9216, 128
    x5 = rnd(B, C, T, HW, 1, seed=94)
    wt = rnd(C, C, 3, 1, 1, seed=95, scale=(3 * C) ** -0.5)
    ref5 = F.conv3d(x5.float(), wt.float(), None, padding=(1, 0, 0))
    rows = lambda t5: t5.permute(0, 2, 3, 4, 1).reshape(B * T * HW, C).contiguous()
    close(ops.conv_temporal(rows(x5), B, T, HW, ops.pack_conv_temporal(wt)), rows(ref5), 3e-3, what="many-tile conv_temporal")


def test_softmax_rows(ops):
    x = rnd(200, 1000, seed=71, dtype=torch.float32, scale=20.0)
    close(ops.softmax_rows(x, 0.044), torch.softmax(x * 0.044, -1), 1e-4, rtol=2e-3, what="softmax_rows")


@pytest.mark.parametrize("M,K,N,res", [(777, 320, 320, True), (4096, 1280, 640, True), (300, 512, 512, False)])
def test_linear_emits_layernorm_statistics_of_its_output(ops, M, K, N, res):
    """ops.linear(..., ln_out=True): the (mean, rstd) the producing GEMM's epilogue gathers equal a statistics pass over the stored
    fp16 output (both use the fp16-rounded values); the output itself is unchanged."""
    x, w = rnd(M, K, seed=41), rnd(N, K, scale=0.05, seed=42)
    b = torch.randn(N, generator=torch.Generator().manual_seed(43)).cuda() * 0.1
    r = rnd(M, N, seed=44) if res else None
    y_ref = ops.linear(x, w, bias=b, res=r)
    y, st = ops.linear(x, w, bias=b, res=r, ln_out=True)
    assert torch.equal(y, y_ref)
    ref = ops.layernorm_stats(y_ref)
    yf = y_ref.float()
    mean, rstd = yf.mean(1), torch.rsqrt(yf.var(1, unbiased=False) + 1e-5)
    assert float((st[:, 0] - mean).abs().max()) < 2e-4 * max(1.0, float(mean.abs().max()))
    assert float(((st[:, 1] - rstd) / rstd).abs().max()) < 2e-4
    assert float((st - ref).abs().max()) < 1e-3


@pytest.mark.parametrize("frames,H,W,Ci,Co", [(3, 9, 16, 64, 64), (2, 18, 32, 320, 160), (2, 36, 64, 128, 96), (1, 5, 7, 32, 32)])
def test_upsample_conv_fused(ops, frames, H, W, Ci, Co):
    """ops.upconv3x3 (four parity sub-convolutions on the small image, strided TMA stores) vs F.interpolate(nearest x2) + conv2d."""
    x = rnd(frames * H * W, Ci, seed=51)
    w = torch.randn(Co, Ci, 3, 3, generator=torch.Generator().manual_seed(52)) * (1.0 / math.sqrt(9 * Ci))
    b = torch.randn(Co, generator=torch.Generator().manual_seed(53)).cuda() * 0.1
    y = ops.upconv3x3(x, frames, H, W, [p.cuda() for p in ops.pack_upconv3x3(w)], bias=b)
    xi = x.float().reshape(frames, H, W, Ci).permute(0, 3, 1, 2)
    ref = F.conv2d(F.interpolate(xi, scale_factor=2, mode="nearest"), w.cuda(), b, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, Co)
    close(y, ref, atol=6e-3, what="upconv3x3")


# ------------------------------------------------------------------ GroupNorm statistics from the producing GEMM's epilogue
def _gn_ref(y, samples, g, b, eps, silu):
    rows, C = y.shape[0] // samples, y.shape[1]
    xr = y.float().reshape(samples, rows, C).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, g, b, eps)
    if silu:
        ref = F.silu(ref)
    return ref.permute(0, 2, 1).reshape(samples * rows, C)


def _force_gn_parts(ops, monkeypatch, mode=2):
    monkeypatch.setattr(ops, "GN_FROM_PRODUCER", mode)
    monkeypatch.setattr(ops, "GN_PARTS_MIN_MB", 0.0)


@pytest.mark.parametrize("frames,H,W,Ci,Co", [(3, 9, 16, 64, 320), (2, 18, 32, 320, 640), (2, 36, 64, 128, 320), (3, 72, 128, 64, 320),
                                               (5, 9, 16, 320, 1280)])
def test_groupnorm_from_conv3x3_partial_sums(ops, monkeypatch, frames, H, W, Ci, Co):
    """conv3x3(gn_out=True) leaves per-(32-row block, chunk, piece) sums; groupnorm() on that tensor (4-D: one sample per frame, and
    5-D: one sample over all frames) skips its statistics pass and must equal the GroupNorm of the stored output."""
    _force_gn_parts(ops, monkeypatch)
    x = rnd(frames * H * W, Ci, seed=61)
    w = ops.pack_conv3x3(torch.randn(Co, Ci, 3, 3, generator=torch.Generator().manual_seed(62)) * (2.0 / math.sqrt(9 * Ci))).cuda()
    bias = torch.randn(Co, generator=torch.Generator().manual_seed(63)).cuda()
    r = rnd(frames * H * W, Co, seed=64)
    y_ref = ops.conv3x3(x, frames, H, W, w, bias=bias, res=r)
    y = ops.conv3x3(x, frames, H, W, w, bias=bias, res=r, gn_out=True)
    assert torch.equal(y, y_ref) and ops.gn_part_of(y) is not None
    g, b = rnd(Co, seed=65, dtype=torch.float32), rnd(Co, seed=66, dtype=torch.float32)
    n0 = ops.gn_from_parts_calls
    out4 = ops.groupnorm(y, frames, g, b, 1e-5, True)
    assert ops.gn_from_parts_calls - n0 == 1, "expected finalize + apply (the partial-sum path), not the statistics-pass kernel"
    close(out4, _gn_ref(y_ref, frames, g, b, 1e-5, True), 3e-3, what="4-D from parts")
    assert torch.equal(out4, ops.groupnorm(y, frames, g, b, 1e-5, True)), "not deterministic"
    out5 = ops.groupnorm(y, 1, g, b, 1e-6, False)
    close(out5, _gn_ref(y_ref, 1, g, b, 1e-6, False), 3e-3, what="5-D from parts")
    # the path without the producer's sums gives the same result up to fp32 summation order
    assert float((out4.float() - ops.groupnorm(y_ref, frames, g, b, 1e-5, True).float()).abs().max()) < 4e-3


@pytest.mark.parametrize("B,T,HW,C", [(2, 5, 576, 320), (1, 7, 144, 640), (2, 4, 2304, 320), (1, 3, 96, 1280)])
def test_groupnorm_from_temporal_conv_and_linear_partial_sums(ops, monkeypatch, B, T, HW, C):
    """Producers in the linear row geometry (temporal conv: Z = B slabs of T*HW rows; 1x1 linear: one slab): consumers are the 5-D
    GroupNorm (sample = batch element) and the 4-D GroupNorm (sample = frame, HW % 32 == 0; otherwise the statistics-pass path)."""
    _force_gn_parts(ops, monkeypatch)
    M = B * T * HW
    x = rnd(M, C, seed=71)
    w3 = ops.pack_conv_temporal(torch.randn(C, C, 3, 1, 1, generator=torch.Generator().manual_seed(72)) * (2.0 / math.sqrt(3 * C))).cuda()
    y = ops.conv_temporal(x, B, T, HW, w3, bias=None, res=x, gn_out=True)
    y_ref = ops.conv_temporal(x, B, T, HW, w3, bias=None, res=x)
    assert torch.equal(y, y_ref)
    g, b = rnd(C, seed=73, dtype=torch.float32), rnd(C, seed=74, dtype=torch.float32)
    close(ops.groupnorm(y, B, g, b, 1e-5, True), _gn_ref(y_ref, B, g, b, 1e-5, True), 3e-3, what="5-D after temporal conv")
    n0 = ops.gn_from_parts_calls
    out = ops.groupnorm(y, B * T, g, b, 1e-6, False)
    assert (ops.gn_from_parts_calls - n0 == 1) == (HW % 32 == 0)
    close(out, _gn_ref(y_ref, B * T, g, b, 1e-6, False), 3e-3, what="4-D after temporal conv")
    wl = rnd(C, C, seed=75, scale=2.0 * C ** -0.5)
    z = ops.linear(x, wl, res=y_ref, gn_out=True)
    z_ref = ops.linear(x, wl, res=y_ref)
    assert torch.equal(z, z_ref) and ops.gn_part_of(z) is not None
    close(ops.groupnorm(z, B, g, b, 1e-5, True), _gn_ref(z_ref, B, g, b, 1e-5, True), 3e-3, what="5-D after linear")
    close(ops.groupnorm(z, B * T, g, b, 1e-5, True), _gn_ref(z_ref, B * T, g, b, 1e-5, True), 3e-3, what="4-D after linear")


@pytest.mark.parametrize("C1,C2", [(320, 320), (640, 320), (640, 640), (1280, 640), (1280, 1280)])
def test_groupnorm_concat_from_partial_sums(ops, monkeypatch, C1, C2):
    """The skip-concat GroupNorm of the output blocks: both sources carry their producers' sums; groups of (C1 + C2) / 32 = 20 / 30 / 40 /
    60 / 80 channels are assembled from the 10-channel sub-groups of the two sources (a group may straddle the concat boundary)."""
    _force_gn_parts(ops, monkeypatch)
    frames, H, W = 3, 18, 32
    M = frames * H * W
    xa, xb = rnd(M, 64, seed=81), rnd(M, 64, seed=82)
    wa = rnd(C1, 64, seed=83, scale=0.3)
    wb = ops.pack_conv3x3(torch.randn(C2, 64, 3, 3, generator=torch.Generator().manual_seed(84)) * 0.1).cuda()
    a = ops.linear(xa, wa, gn_out=True)
    s = ops.conv3x3(xb, frames, H, W, wb, gn_out=True)
    C = C1 + C2
    g, b = rnd(C, seed=85, dtype=torch.float32), rnd(C, seed=86, dtype=torch.float32)
    n0 = ops.gn_from_parts_calls
    out = ops.groupnorm(a, frames, g, b, 1e-5, True, x2=s)
    assert ops.gn_from_parts_calls - n0 == 1
    ref = _gn_ref(torch.cat([a, s], 1), frames, g, b, 1e-5, True)
    close(out, ref, 3e-3, what="concat from parts")
    a2 = a.clone()                                          # a source without sums -> the statistics-pass kernel
    close(ops.groupnorm(a2, frames, g, b, 1e-5, True, x2=s), ref, 3e-3, what="concat fallback")


def test_gemm_output_unchanged_by_gn_out_large_and_small(ops, monkeypatch):
    """Large and small tile counts (several persistent rounds / fewer tiles than SMs): the records of both are consumed."""
    _force_gn_parts(ops, monkeypatch)
    for M, K, N in ((128 * 301, 320, 320), (128 * 3 + 40, 640, 640), (40000, 1280, 320)):
        x, w = rnd(M, K, seed=91), rnd(N, K, seed=92, scale=2.0 * K ** -0.5)
        y = ops.linear(x, w, gn_out=True)
        assert torch.equal(y, ops.linear(x, w))
        g, b = rnd(N, seed=93, dtype=torch.float32), rnd(N, seed=94, dtype=torch.float32)
        close(ops.groupnorm(y, 1, g, b, 1e-5, False), _gn_ref(y, 1, g, b, 1e-5, False), 3e-3, what=f"M={M}")
