"""Oracle for the ViewCrafter DDIM-denoise hot path.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference``
legs of ``bench.py`` may import this file.  Nothing in ``viewcrafter_b200/`` does.

This is a functional (state-dict driven, fp32, plain-torch) restatement of the reference
algorithm.  It is device-agnostic: on the CPU it is the checker of the small parity cases; on a
CUDA device (tensors + state dict moved there, TF32 off -- see ``exact_fp32``) it is the checker
at the BASELINE.json sizes (25x4x40x64, 25x4x72x128) where a CPU run takes minutes, and, run under
``torch.autocast(fp16)`` with ``attention_mode("sdpa")``, it is the stand-in for "the unmodified
reference in PyTorch eager on the same GPU" (viewcrafter.py:98 runs the reference under autocast;
attention.py:175-190 uses xformers' fused attention when present).  Every function cites the reference file:line (paths relative to the upstream
repo root) it follows.  The block structure is recovered from the *state-dict keys* (which
are the reference's load-bearing interface, SURVEY.md Appendix B), not from a copy of the
reference constructor.

Parity pinning: the reference ships no tests / golden vectors for this path ("parity
unpinned" by the reference itself).  We pin this oracle instead against outputs of the
unmodified reference modules imported from /root/reference in the build container:
``oracle/make_golden.py`` generates ``tests/golden/*.npz`` and ``tests/test_oracle_golden.py``
checks this file against them (and, when /root/reference is present, against the live
reference modules).
"""
from __future__ import annotations

import contextlib
import math
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]

_ATTN = {"mode": "naive", "chunk_bytes": 2 << 30}


@contextlib.contextmanager
def attention_mode(mode: str):
    """'naive' = the in-tree softmax(QK^T)V of attention.py:103-120 (evaluated in batch chunks so the score matrix
    stays below 2 GiB; rows are independent, so the result is the unchunked one).  'sdpa' = one fused
    scaled_dot_product_attention call per attention, the math xformers.ops.memory_efficient_attention performs in
    the reference's efficient_forward (attention.py:146-190)."""
    old = _ATTN["mode"]
    _ATTN["mode"] = mode
    try:
        yield
    finally:
        _ATTN["mode"] = old


@contextlib.contextmanager
def exact_fp32():
    """fp32 means fp32: no TF32 in cuBLAS / cuDNN while the oracle runs on a CUDA device."""
    a, b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    prec = torch.get_float32_matmul_precision()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = a, b
        torch.set_float32_matmul_precision(prec)


# --------------------------------------------------------------------------------------
# schedule / scalar tables  (lvdm/models/utils_diffusion.py, lvdm/models/ddpm3d.py)
# --------------------------------------------------------------------------------------
def timestep_embedding(timesteps: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    """cos||sin sinusoid, lvdm/models/utils_diffusion.py:8-28."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=torch.float32) / half).to(timesteps.device)
    args = timesteps[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


def make_beta_schedule_linear(n: int, linear_start: float, linear_end: float) -> np.ndarray:
    """'linear' branch of lvdm/models/utils_diffusion.py:31-35 (float64)."""
    return (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n, dtype=torch.float64) ** 2).numpy()


def rescale_zero_terminal_snr(betas: np.ndarray) -> np.ndarray:
    """lvdm/models/utils_diffusion.py:112-144."""
    ab_sqrt = np.sqrt(np.cumprod(1.0 - betas, axis=0))
    first, last = ab_sqrt[0].copy(), ab_sqrt[-1].copy()
    ab_sqrt = ab_sqrt - last
    ab_sqrt = ab_sqrt * (first / (first - last))
    ab = ab_sqrt ** 2
    alphas = np.concatenate([ab[0:1], ab[1:] / ab[:-1]])
    return 1 - alphas


def model_schedule(timesteps=1000, linear_start=0.00085, linear_end=0.012, zero_snr=True,
                   base_scale=0.3, turning_step=400) -> Dict[str, torch.Tensor]:
    """Buffers the sampler reads from the model: lvdm/models/ddpm3d.py:123-150 and :522-527."""
    betas = make_beta_schedule_linear(timesteps, linear_start, linear_end)
    if zero_snr:
        betas = rescale_zero_terminal_snr(betas)
    ac = np.cumprod(1.0 - betas, axis=0)
    ac_prev = np.append(1.0, ac[:-1])
    f32 = lambda a: torch.tensor(a, dtype=torch.float32)
    scale_arr = np.concatenate((np.linspace(1.0, base_scale, turning_step), np.full(timesteps, base_scale)))
    return dict(betas=f32(betas), alphas_cumprod=f32(ac), alphas_cumprod_prev=f32(ac_prev),
                sqrt_alphas_cumprod=f32(np.sqrt(ac)), sqrt_one_minus_alphas_cumprod=f32(np.sqrt(1.0 - ac)),
                scale_arr=f32(scale_arr))


def make_ddim_timesteps(method: str, n_ddim: int, n_ddpm: int) -> np.ndarray:
    """lvdm/models/utils_diffusion.py:56-76."""
    if method == "uniform":
        c = n_ddpm // n_ddim
        return np.asarray(list(range(0, n_ddpm, c))) + 1
    if method == "uniform_trailing":
        c = n_ddpm / n_ddim
        return np.flip(np.round(np.arange(n_ddpm, 0, -c))).astype(np.int64) - 1
    if method == "quad":
        return ((np.linspace(0, np.sqrt(n_ddpm * .8), n_ddim)) ** 2).astype(int) + 1
    raise NotImplementedError(method)


def ddim_tables(sched: Dict[str, torch.Tensor], S: int, method: str, eta: float, fixed_prev_scale: bool = True):
    """DDIMSampler.make_schedule, lvdm/models/samplers/ddim.py:24-59.

    Reproduces the dtype quirks: alphas come from the model's float32 ``alphas_cumprod``;
    sigmas/alphas are torch float32->float64?  No: ``alphacums`` is a float32 torch tensor, so
    ``alphas`` is a float32 tensor, ``alphas_prev`` a numpy float64 array built from python
    floats, and ``sigmas`` a float64 tensor (tensor op with a float64 numpy array promotes).
    """
    ts = make_ddim_timesteps(method, S, sched["alphas_cumprod"].shape[0])
    alphacums = sched["alphas_cumprod"].cpu()
    alphas = alphacums[ts]
    alphas_prev = np.asarray([alphacums[0]] + alphacums[ts[:-1]].tolist())
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    sqrt_1m = np.sqrt(1.0 - alphas)
    scale = sched["scale_arr"][ts]
    head = sched["scale_arr"][0:1] if fixed_prev_scale else scale[0:1]   # ddim.py:35 vs ddim_multiplecond.py:33
    scale_prev = torch.cat([head, scale[:-1]])
    return dict(timesteps=ts, alphas=alphas, alphas_prev=alphas_prev, sigmas=sigmas,
                sqrt_one_minus_alphas=sqrt_1m, scale=scale, scale_prev=scale_prev)


def step_scalars(tab, index: int) -> np.ndarray:
    """The six fp32 scalars p_sample_ddim materialises with torch.full (ddim.py:253-266):
    [a_t, a_prev, sigma_t, sqrt(1-a_t), scale_t, prev_scale_t].  Whatever the source dtype
    (fp32 tensor, numpy float64, float64 tensor) torch.full rounds the value to float32."""
    vals = [tab["alphas"][index], tab["alphas_prev"][index], tab["sigmas"][index],
            tab["sqrt_one_minus_alphas"][index], tab["scale"][index], tab["scale_prev"][index]]
    return np.asarray([torch.full((1,), float(v)).item() for v in vals], dtype=np.float32)


# --------------------------------------------------------------------------------------
# U-Net blocks  (lvdm/modules/networks/openaimodel3d.py, lvdm/modules/attention.py)
# --------------------------------------------------------------------------------------
def _gn(x, sd: SD, p: str, eps: float):
    return F.group_norm(x.float(), 32, sd[p + ".weight"], sd[p + ".bias"], eps)


def _lin(x, sd: SD, p: str):
    return F.linear(x, sd[p + ".weight"], sd.get(p + ".bias"))


def temporal_conv_block(sd: SD, p: str, x5: torch.Tensor) -> torch.Tensor:
    """TemporalConvBlock.forward, openaimodel3d.py:239-279: 4x[GN32(eps 1e-5 over C/32,T,H,W)+SiLU+Conv3d(3,1,1)] + identity."""
    h = x5
    for name, ci in (("conv1", 2), ("conv2", 3), ("conv3", 3), ("conv4", 3)):
        h = F.silu(_gn(h, sd, f"{p}.{name}.0", 1e-5))
        h = F.conv3d(h, sd[f"{p}.{name}.{ci}.weight"], sd[f"{p}.{name}.{ci}.bias"], padding=(1, 0, 0))
    return x5 + h


def res_block(sd: SD, p: str, x: torch.Tensor, emb: torch.Tensor, T: int) -> torch.Tensor:
    """ResBlock._forward, openaimodel3d.py:210-236 (no up/down, no scale-shift norm)."""
    h = F.conv2d(F.silu(_gn(x, sd, p + ".in_layers.0", 1e-5)), sd[p + ".in_layers.2.weight"], sd[p + ".in_layers.2.bias"], padding=1)
    h = h + _lin(F.silu(emb), sd, p + ".emb_layers.1")[:, :, None, None]
    h = F.conv2d(F.silu(_gn(h, sd, p + ".out_layers.0", 1e-5)), sd[p + ".out_layers.3.weight"], sd[p + ".out_layers.3.bias"], padding=1)
    if p + ".skip_connection.weight" in sd:
        x = F.conv2d(x, sd[p + ".skip_connection.weight"], sd[p + ".skip_connection.bias"])
    h = x + h
    if p + ".temopral_conv.conv1.0.weight" in sd:
        BT, C, H, W = h.shape
        h5 = h.reshape(BT // T, T, C, H, W).permute(0, 2, 1, 3, 4)
        h5 = temporal_conv_block(sd, p + ".temopral_conv", h5)
        h = h5.permute(0, 2, 1, 3, 4).reshape(BT, C, H, W)
    return h


def _heads(t: torch.Tensor, h: int):
    b, n, c = t.shape
    return t.reshape(b, n, h, c // h).permute(0, 2, 1, 3)          # b h n d


def _attend(q, k, v, scale):
    """naive softmax attention, attention.py:103-120 (see attention_mode)."""
    if _ATTN["mode"] == "sdpa":
        return F.scaled_dot_product_attention(q, k, v, scale=scale)
    b, h, n, _ = q.shape
    per_b = h * n * k.shape[2] * 4
    bs = max(1, _ATTN["chunk_bytes"] // max(per_b, 1))
    if bs >= b:
        sim = torch.einsum("bhid,bhjd->bhij", q, k) * scale
        return torch.einsum("bhij,bhjd->bhid", sim.softmax(dim=-1), v)
    outs = []
    for i in range(0, b, bs):
        sim = torch.einsum("bhid,bhjd->bhij", q[i:i + bs], k[i:i + bs]) * scale
        outs.append(torch.einsum("bhij,bhjd->bhid", sim.softmax(dim=-1), v[i:i + bs]))
    return torch.cat(outs, 0)


def cross_attention(sd: SD, p: str, x: torch.Tensor, ctx: Optional[torch.Tensor], d_head: int = 64, text_len: int = 77):
    """CrossAttention.forward, attention.py:81-144 (no rel-pos, no mask).  ctx=None -> self-attention.
    When the module owns to_k_ip/to_v_ip the context is split text[:77] | image[77:] and the two
    attention outputs are summed with scale 1.0 (attention.py:89-94,128-142)."""
    heads = sd[p + ".to_q.weight"].shape[0] // d_head
    scale = d_head ** -0.5
    q = _heads(F.linear(x, sd[p + ".to_q.weight"]), heads)
    has_ip = (p + ".to_k_ip.weight") in sd
    if ctx is None:
        kv_src = x
    else:
        kv_src = ctx[:, :text_len, :]
    k = _heads(F.linear(kv_src, sd[p + ".to_k.weight"]), heads)
    v = _heads(F.linear(kv_src, sd[p + ".to_v.weight"]), heads)
    out = _attend(q, k, v, scale)
    if has_ip and ctx is not None:
        img = ctx[:, text_len:, :]
        k_ip = _heads(F.linear(img, sd[p + ".to_k_ip.weight"]), heads)
        v_ip = _heads(F.linear(img, sd[p + ".to_v_ip.weight"]), heads)
        out = out + 1.0 * _attend(q, k_ip, v_ip, scale)
    b, h, n, d = out.shape
    out = out.permute(0, 2, 1, 3).reshape(b, n, h * d)
    return _lin(out, sd, p + ".to_out.0")


def _ln(x, sd: SD, p: str):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-5)


def feed_forward(sd: SD, p: str, x):
    """FeedForward with GEGLU, attention.py:415-442 (exact-erf GELU)."""
    a, gate = _lin(x, sd, p + ".net.0.proj").chunk(2, dim=-1)
    return _lin(a * F.gelu(gate), sd, p + ".net.2")


def basic_transformer_block(sd: SD, p: str, x, ctx):
    """BasicTransformerBlock._forward, attention.py:242-246.  attn1 is always self-attention;
    attn2 uses ctx (None for the temporal transformer => self-attention again)."""
    x = cross_attention(sd, p + ".attn1", _ln(x, sd, p + ".norm1"), None) + x
    x = cross_attention(sd, p + ".attn2", _ln(x, sd, p + ".norm2"), ctx) + x
    x = feed_forward(sd, p + ".ff", _ln(x, sd, p + ".norm3")) + x
    return x


def spatial_transformer(sd: SD, p: str, x: torch.Tensor, ctx: torch.Tensor) -> torch.Tensor:
    """SpatialTransformer.forward (use_linear=True), attention.py:294-310."""
    BT, C, H, W = x.shape
    h = _gn(x, sd, p + ".norm", 1e-6)
    h = h.permute(0, 2, 3, 1).reshape(BT, H * W, C)
    h = _lin(h, sd, p + ".proj_in")
    h = basic_transformer_block(sd, p + ".transformer_blocks.0", h, ctx)
    h = _lin(h, sd, p + ".proj_out")
    return h.reshape(BT, H, W, C).permute(0, 3, 1, 2) + x


def temporal_transformer(sd: SD, p: str, x: torch.Tensor, T: int) -> torch.Tensor:
    """TemporalTransformer.forward (only_self_att, no mask), attention.py:365-412.
    proj_in/out are nn.Linear (use_linear) or Conv1d k=1 (init_attn) -- same math."""
    BT, C, H, W = x.shape
    B = BT // T
    x5 = x.reshape(B, T, C, H, W).permute(0, 2, 1, 3, 4)                      # b c t h w
    h = _gn(x5, sd, p + ".norm", 1e-6)                                       # stats over (C/32, T, H, W)
    h = h.permute(0, 3, 4, 2, 1).reshape(B * H * W, T, C)                    # (b h w) t c
    w_in, w_out = sd[p + ".proj_in.weight"], sd[p + ".proj_out.weight"]
    h = F.linear(h, w_in.reshape(w_in.shape[0], w_in.shape[1]), sd[p + ".proj_in.bias"])
    h = basic_transformer_block(sd, p + ".transformer_blocks.0", h, None)
    h = F.linear(h, w_out.reshape(w_out.shape[0], w_out.shape[1]), sd[p + ".proj_out.bias"])
    h = h.reshape(B, H, W, T, C).permute(0, 4, 3, 1, 2)                      # b c t h w
    out = h + x5
    return out.permute(0, 2, 1, 3, 4).reshape(BT, C, H, W)


def _run_stage(sd: SD, p: str, h, emb, ctx, T):
    """TimestepEmbedSequential dispatch (openaimodel3d.py:36-48), structure recovered from keys."""
    j = 0
    while True:
        q = f"{p}.{j}"
        if q + ".in_layers.0.weight" in sd:
            h = res_block(sd, q, h, emb, T)
        elif q + ".transformer_blocks.0.attn2.to_k_ip.weight" in sd:
            h = spatial_transformer(sd, q, h, ctx)
        elif q + ".transformer_blocks.0.attn1.to_q.weight" in sd:
            h = temporal_transformer(sd, q, h, T)
        elif q + ".op.weight" in sd:                                         # Downsample, :51-77
            h = F.conv2d(h, sd[q + ".op.weight"], sd[q + ".op.bias"], stride=2, padding=1)
        elif q + ".conv.weight" in sd:                                       # Upsample, :80-106
            h = F.interpolate(h, scale_factor=2, mode="nearest")
            h = F.conv2d(h, sd[q + ".conv.weight"], sd[q + ".conv.bias"], padding=1)
        elif q + ".weight" in sd and sd[q + ".weight"].dim() == 4:           # input conv
            h = F.conv2d(h, sd[q + ".weight"], sd[q + ".bias"], padding=1)
        else:
            break
        j += 1
    return h


def unet_forward(sd: SD, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor,
                 fs: Optional[torch.Tensor] = None, default_fs: int = 10) -> torch.Tensor:
    """UNetModel.forward, openaimodel3d.py:548-603.  x [B,Cin,T,H,W] -> [B,Cout,T,H,W]."""
    B, _, T, H, W = x.shape
    mc = sd["time_embed.0.weight"].shape[1]
    emb = _lin(F.silu(_lin(timestep_embedding(timesteps, mc), sd, "time_embed.0")), sd, "time_embed.2")
    if context.shape[1] == 77 + T * 16:                                      # :556-560 (true for T=16)
        txt = context[:, :77].repeat_interleave(T, dim=0)
        img = context[:, 77:].reshape(B, T, 16, -1).reshape(B * T, 16, -1)
        ctx = torch.cat([txt, img], dim=1)
    else:
        ctx = context.repeat_interleave(T, dim=0)
    emb = emb.repeat_interleave(T, dim=0)
    if "fps_embedding.0.weight" in sd:
        if fs is None:
            fs = torch.tensor([default_fs] * B, dtype=torch.long, device=x.device)
        fe = _lin(F.silu(_lin(timestep_embedding(fs, mc), sd, "fps_embedding.0")), sd, "fps_embedding.2")
        emb = emb + fe.repeat_interleave(T, dim=0)
    h = x.permute(0, 2, 1, 3, 4).reshape(B * T, -1, H, W).float()
    hs: List[torch.Tensor] = []
    i = 0
    while f"input_blocks.{i}.0.weight" in sd or f"input_blocks.{i}.0.in_layers.0.weight" in sd or f"input_blocks.{i}.0.op.weight" in sd:
        h = _run_stage(sd, f"input_blocks.{i}", h, emb, ctx, T)
        if i == 0 and "init_attn.0.norm.weight" in sd:
            h = temporal_transformer(sd, "init_attn.0", h, T)
        hs.append(h)
        i += 1
    h = _run_stage(sd, "middle_block", h, emb, ctx, T)
    i = 0
    while f"output_blocks.{i}.0.in_layers.0.weight" in sd:
        h = torch.cat([h, hs.pop()], dim=1)
        h = _run_stage(sd, f"output_blocks.{i}", h, emb, ctx, T)
        i += 1
    y = F.conv2d(F.silu(_gn(h, sd, "out.0", 1e-5)), sd["out.2.weight"], sd["out.2.bias"], padding=1)
    return y.reshape(B, T, -1, H, W).permute(0, 2, 1, 3, 4)


# --------------------------------------------------------------------------------------
# VAE decoder  (lvdm/modules/networks/ae_modules.py, lvdm/models/autoencoder.py)
# --------------------------------------------------------------------------------------
def _swish(x):
    return x * torch.sigmoid(x)


def vae_resnet_block(sd: SD, p: str, x):
    """ae_modules.ResnetBlock.forward (temb=None), ae_modules.py:190-210; GN eps 1e-6."""
    h = F.conv2d(_swish(_gn(x, sd, p + ".norm1", 1e-6)), sd[p + ".conv1.weight"], sd[p + ".conv1.bias"], padding=1)
    h = F.conv2d(_swish(_gn(h, sd, p + ".norm2", 1e-6)), sd[p + ".conv2.weight"], sd[p + ".conv2.bias"], padding=1)
    if p + ".nin_shortcut.weight" in sd:
        x = F.conv2d(x, sd[p + ".nin_shortcut.weight"], sd[p + ".nin_shortcut.bias"])
    return x + h


def vae_attn_block(sd: SD, p: str, x):
    """ae_modules.AttnBlock.forward, ae_modules.py:53-78: single head, d=C, scale C^-0.5."""
    B, C, H, W = x.shape
    h = _gn(x, sd, p + ".norm", 1e-6)
    q = F.conv2d(h, sd[p + ".q.weight"], sd[p + ".q.bias"]).reshape(B, C, H * W).permute(0, 2, 1)
    k = F.conv2d(h, sd[p + ".k.weight"], sd[p + ".k.bias"]).reshape(B, C, H * W)
    v = F.conv2d(h, sd[p + ".v.weight"], sd[p + ".v.bias"]).reshape(B, C, H * W)
    w = torch.softmax(torch.bmm(q, k) * (int(C) ** -0.5), dim=2)
    o = torch.bmm(v, w.permute(0, 2, 1)).reshape(B, C, H, W)
    return x + F.conv2d(o, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"])


def vae_decode(sd: SD, z: torch.Tensor) -> torch.Tensor:
    """AutoencoderKL.decode (autoencoder.py:104-107) -> Decoder.forward (ae_modules.py:539-578).
    sd keys are relative to the autoencoder ("post_quant_conv.*", "decoder.*")."""
    z = F.conv2d(z, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
    d = "decoder"
    h = F.conv2d(z, sd[d + ".conv_in.weight"], sd[d + ".conv_in.bias"], padding=1)
    h = vae_resnet_block(sd, d + ".mid.block_1", h)
    h = vae_attn_block(sd, d + ".mid.attn_1", h)
    h = vae_resnet_block(sd, d + ".mid.block_2", h)
    n_levels = 0
    while f"{d}.up.{n_levels}.block.0.norm1.weight" in sd:
        n_levels += 1
    for lvl in reversed(range(n_levels)):
        b = 0
        while f"{d}.up.{lvl}.block.{b}.norm1.weight" in sd:
            h = vae_resnet_block(sd, f"{d}.up.{lvl}.block.{b}", h)
            if f"{d}.up.{lvl}.attn.{b}.norm.weight" in sd:
                h = vae_attn_block(sd, f"{d}.up.{lvl}.attn.{b}", h)
            b += 1
        if f"{d}.up.{lvl}.upsample.conv.weight" in sd:
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = F.conv2d(h, sd[f"{d}.up.{lvl}.upsample.conv.weight"], sd[f"{d}.up.{lvl}.upsample.conv.bias"], padding=1)
    h = _swish(_gn(h, sd, d + ".norm_out", 1e-6))
    return F.conv2d(h, sd[d + ".conv_out.weight"], sd[d + ".conv_out.bias"], padding=1)


def vae_encode_moments(sd: SD, x: torch.Tensor) -> torch.Tensor:
    """AutoencoderKL.encode up to the moments (autoencoder.py:97-100) -> Encoder.forward (ae_modules.py:430-463);
    Downsample = zero-pad right/bottom by one, then 3x3 stride-2 conv without padding (ae_modules.py:102-106).
    sd keys are relative to the autoencoder ("encoder.*", "quant_conv.*").  Returns [N, 2*embed_dim, h, w]."""
    e = "encoder"
    h = F.conv2d(x, sd[e + ".conv_in.weight"], sd[e + ".conv_in.bias"], padding=1)
    lvl = 0
    while f"{e}.down.{lvl}.block.0.norm1.weight" in sd:
        b = 0
        while f"{e}.down.{lvl}.block.{b}.norm1.weight" in sd:
            h = vae_resnet_block(sd, f"{e}.down.{lvl}.block.{b}", h)
            if f"{e}.down.{lvl}.attn.{b}.norm.weight" in sd:
                h = vae_attn_block(sd, f"{e}.down.{lvl}.attn.{b}", h)
            b += 1
        if f"{e}.down.{lvl}.downsample.conv.weight" in sd:
            h = F.pad(h, (0, 1, 0, 1), mode="constant", value=0)
            h = F.conv2d(h, sd[f"{e}.down.{lvl}.downsample.conv.weight"], sd[f"{e}.down.{lvl}.downsample.conv.bias"], stride=2)
        lvl += 1
    h = vae_resnet_block(sd, e + ".mid.block_1", h)
    h = vae_attn_block(sd, e + ".mid.attn_1", h)
    h = vae_resnet_block(sd, e + ".mid.block_2", h)
    h = _swish(_gn(h, sd, e + ".norm_out", 1e-6))
    h = F.conv2d(h, sd[e + ".conv_out.weight"], sd[e + ".conv_out.bias"], padding=1)
    return F.conv2d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])


def posterior_sample(moments: torch.Tensor, noise: torch.Tensor) -> torch.Tensor:
    """DiagonalGaussianDistribution.__init__ + sample (distributions.py:24-40): logvar clamped to [-30, 20]."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    return mean + torch.exp(0.5 * logvar) * noise


def encode_first_stage(sd: SD, x5: torch.Tensor, noises: List[torch.Tensor], scale_factor: float = 0.18215) -> torch.Tensor:
    """LatentDiffusion.encode_first_stage with perframe_ae + get_first_stage_encoding (ddpm3d.py:611-644): one posterior
    sample per frame (noises[i] is the randn the i-th frame's DiagonalGaussianDistribution.sample draws), times scale_factor."""
    B, C, T, H, W = x5.shape
    x = x5.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)
    outs = [scale_factor * posterior_sample(vae_encode_moments(sd, x[i:i + 1]), noises[i]) for i in range(x.shape[0])]
    r = torch.cat(outs, dim=0)
    return r.reshape(B, T, r.shape[1], r.shape[2], r.shape[3]).permute(0, 2, 1, 3, 4)


def decode_first_stage(sd: SD, z5: torch.Tensor, scale_factor: float = 0.18215) -> torch.Tensor:
    """LatentDiffusion.decode_core with perframe_ae, ddpm3d.py:646-667."""
    B, C, T, H, W = z5.shape
    z = z5.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)
    outs = [vae_decode(sd, 1.0 / scale_factor * z[i:i + 1]) for i in range(z.shape[0])]
    r = torch.cat(outs, dim=0)
    return r.reshape(B, T, r.shape[1], r.shape[2], r.shape[3]).permute(0, 2, 1, 3, 4)


# --------------------------------------------------------------------------------------
# image-context projector  (lvdm/modules/encoders/resampler.py) -- SURVEY.md 8(f) rank f3
# --------------------------------------------------------------------------------------
def perceiver_attention(sd: SD, p: str, x: torch.Tensor, latents: torch.Tensor, heads: int, dim_head: int = 64) -> torch.Tensor:
    """PerceiverAttention.forward, resampler.py:62-94: queries from the latents, keys/values from cat(image tokens,
    latents); q and k are each scaled by dim_head**-0.25 before the product; softmax in fp32."""
    x = F.layer_norm(x, (x.shape[-1],), sd[p + ".norm1.weight"], sd[p + ".norm1.bias"])
    latents = F.layer_norm(latents, (latents.shape[-1],), sd[p + ".norm2.weight"], sd[p + ".norm2.bias"])
    b, l, _ = latents.shape
    q = F.linear(latents, sd[p + ".to_q.weight"])
    k, v = F.linear(torch.cat((x, latents), dim=-2), sd[p + ".to_kv.weight"]).chunk(2, dim=-1)
    split = lambda t: t.view(b, t.shape[1], heads, -1).transpose(1, 2)
    q, k, v = split(q), split(k), split(v)
    scale = 1 / math.sqrt(math.sqrt(dim_head))
    w = torch.softmax(((q * scale) @ (k * scale).transpose(-2, -1)).float(), dim=-1)
    out = (w @ v).permute(0, 2, 1, 3).reshape(b, l, -1)
    return F.linear(out, sd[p + ".to_out.weight"])


def resampler_forward(sd: SD, x: torch.Tensor, heads: int, dim_head: int = 64) -> torch.Tensor:
    """Resampler.forward, resampler.py:134-145: learned latents (num_queries * video_length of them) attend to the
    projected CLIP tokens through ``depth`` (PerceiverAttention, FeedForward) pairs, each with a residual;
    FeedForward = LayerNorm, Linear(no bias), GELU(erf), Linear(no bias) (resampler.py:27-34)."""
    latents = sd["latents"].repeat(x.shape[0], 1, 1)
    x = F.linear(x, sd["proj_in.weight"], sd["proj_in.bias"])
    depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("layers."))
    for i in range(depth):
        latents = perceiver_attention(sd, f"layers.{i}.0", x, latents, heads, dim_head) + latents
        f = f"layers.{i}.1"
        h = F.layer_norm(latents, (latents.shape[-1],), sd[f + ".0.weight"], sd[f + ".0.bias"])
        h = F.linear(F.gelu(F.linear(h, sd[f + ".1.weight"])), sd[f + ".3.weight"])
        latents = h + latents
    latents = F.linear(latents, sd["proj_out.weight"], sd["proj_out.bias"])
    return F.layer_norm(latents, (latents.shape[-1],), sd["norm_out.weight"], sd["norm_out.bias"])


# --------------------------------------------------------------------------------------
# DDIM sampler  (lvdm/models/samplers/ddim.py)
# --------------------------------------------------------------------------------------
def rescale_noise_cfg(noise_cfg, noise_pred_text, guidance_rescale):
    """utils_diffusion.py:147-158 (unbiased std over all non-batch dims)."""
    dims = list(range(1, noise_pred_text.ndim))
    std_text = noise_pred_text.std(dim=dims, keepdim=True)
    std_cfg = noise_cfg.std(dim=dims, keepdim=True)
    return guidance_rescale * (noise_cfg * (std_text / std_cfg)) + (1 - guidance_rescale) * noise_cfg


def ddim_update(x, v_cond, v_uncond, sc: np.ndarray, sqrt_ac_t: float, sqrt_1mac_t: float,
                noise, cfg_scale: float, guidance_rescale: float, v_uncond_img=None, cfg_img: float = 0.0):
    """Everything in p_sample_ddim after the two apply_model calls, ddim.py:228-281, v-parameterisation
    (ddpm3d.py:239-251).  ``sc`` = step_scalars(...) = [a_t, a_prev, sigma_t, sqrt(1-a_t), scale_t, prev_scale_t];
    sqrt_ac_t / sqrt_1mac_t are the model buffers gathered by the *timestep* t."""
    if v_uncond is None or cfg_scale == 1.0:
        out = v_cond
    else:
        if v_uncond_img is None:
            out = v_uncond + cfg_scale * (v_cond - v_uncond)
        else:       # three-way CFG, ddim_multiplecond.py:227-233
            out = v_uncond + cfg_img * (v_uncond_img - v_uncond) + cfg_scale * (v_cond - v_uncond_img)
        if guidance_rescale > 0.0:
            out = rescale_noise_cfg(out, v_cond, guidance_rescale)
    f = lambda s: torch.tensor(float(s), dtype=torch.float32)
    e_t = f(sqrt_ac_t) * out + f(sqrt_1mac_t) * x
    pred_x0 = f(sqrt_ac_t) * x - f(sqrt_1mac_t) * out
    a_prev, sigma_t = f(sc[1]), f(sc[2])
    pred_x0 = pred_x0 * (f(sc[5]) / f(sc[4]))
    dir_xt = (1.0 - a_prev - sigma_t ** 2).sqrt() * e_t
    x_prev = a_prev.sqrt() * pred_x0 + dir_xt + sigma_t * noise
    return x_prev, pred_x0


def ddim_sample(model_fn, sched, shape, S: int, cond, uncond, x_T: torch.Tensor, noises: List[torch.Tensor],
                eta=1.0, cfg_scale=7.5, guidance_rescale=0.7, method="uniform_trailing", log_every_t=100,
                use_dynamic_rescale=True, fixed_prev_scale=True, uncond_img=None, cfg_img=None):
    """DDIMSampler.sample + ddim_sampling loop, ddim.py:61-205.  ``model_fn(x, t_long, cond)`` plays
    model.apply_model; ``noises[i]`` is the i-th per-step randn draw (the reference draws it with
    torch.randn at ddim.py:275; the oracle takes it as an input so both sides see identical noise).
    ``uncond_img`` (+ ``fixed_prev_scale=False``) gives the three-way-CFG sampler of ddim_multiplecond.py:209-287
    (``cfg_img`` defaults to ``cfg_scale`` like :222-223)."""
    tab = ddim_tables(sched, S, method, eta, fixed_prev_scale)
    if not use_dynamic_rescale:
        tab["scale"] = torch.ones(S); tab["scale_prev"] = torch.ones(S)
    img = x_T
    inter = {"x_inter": [img], "pred_x0": [img]}
    order = np.flip(tab["timesteps"])
    for i, step in enumerate(order):
        index = S - i - 1
        ts = torch.full((shape[0],), int(step), dtype=torch.long, device=img.device)
        v_c = model_fn(img, ts, cond)
        v_u = model_fn(img, ts, uncond) if (uncond is not None and cfg_scale != 1.0) else None
        v_i = model_fn(img, ts, uncond_img) if (uncond_img is not None and v_u is not None) else None
        sc = step_scalars(tab, index)
        img, pred_x0 = ddim_update(img, v_c, v_u, sc, sched["sqrt_alphas_cumprod"][int(step)].item(),
                                   sched["sqrt_one_minus_alphas_cumprod"][int(step)].item(), noises[i],
                                   cfg_scale, guidance_rescale, v_uncond_img=v_i,
                                   cfg_img=cfg_scale if cfg_img is None else cfg_img)
        if index % log_every_t == 0 or index == S - 1:
            inter["x_inter"].append(img); inter["pred_x0"].append(pred_x0)
    return img, inter
