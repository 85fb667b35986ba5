"""Independent restatements of FIFO-Diffusion diagonal denoising for the tests: the per-frame-timestep U-Net assembled from the unchanged
fp32 oracle's pieces, a float64 per-frame DDIM update, and the FIFO loop by its definition (INTEGRATION.md "Long clips: FIFO diagonal
denoising")."""
from __future__ import annotations

from typing import List

import torch
import torch.nn.functional as F

from tests.test_dpm_solver_cpu import dpm_update_f64


def unet_forward_frames(sd, x, timesteps, context, fs=None, default_fs=10):
    """oracle.lvdm_oracle.unet_forward with timesteps [B] or [B, T]: the time embedding runs on one timestep per (sample, frame) and
    fs is repeated per frame; everything after the embeddings is the oracle's own stage code."""
    from oracle import lvdm_oracle as O
    B, _, T, H, W = x.shape
    ts = timesteps.reshape(B, -1).expand(B, T).reshape(-1)
    mc = sd["time_embed.0.weight"].shape[1]
    emb = O._lin(F.silu(O._lin(O.timestep_embedding(ts, mc), sd, "time_embed.0")), sd, "time_embed.2")        # [B*T]
    if context.shape[1] == 77 + T * 16:
        txt = context[:, :77].repeat_interleave(T, dim=0)
        img = context[:, 77:].reshape(B, T, 16, -1).reshape(B * T, 16, -1)
        ctx = torch.cat([txt, img], dim=1)
    else:
        ctx = context.repeat_interleave(T, dim=0)
    if "fps_embedding.0.weight" in sd:
        if fs is None:
            fs = torch.tensor([default_fs] * B, dtype=torch.long, device=x.device)
        fe = O._lin(F.silu(O._lin(O.timestep_embedding(fs, mc), sd, "fps_embedding.0")), sd, "fps_embedding.2")
        emb = emb + fe.repeat_interleave(T, dim=0)
    h = x.permute(0, 2, 1, 3, 4).reshape(B * T, -1, H, W).float()
    hs: List[torch.Tensor] = []
    i = 0
    while f"input_blocks.{i}.0.weight" in sd or f"input_blocks.{i}.0.in_layers.0.weight" in sd or f"input_blocks.{i}.0.op.weight" in sd:
        h = O._run_stage(sd, f"input_blocks.{i}", h, emb, ctx, T)
        if i == 0 and "init_attn.0.norm.weight" in sd:
            h = O.temporal_transformer(sd, "init_attn.0", h, T)
        hs.append(h)
        i += 1
    h = O._run_stage(sd, "middle_block", h, emb, ctx, T)
    i = 0
    while f"output_blocks.{i}.0.in_layers.0.weight" in sd:
        h = torch.cat([h, hs.pop()], dim=1)
        h = O._run_stage(sd, f"output_blocks.{i}", h, emb, ctx, T)
        i += 1
    y = F.conv2d(F.silu(O._gn(h, sd, "out.0", 1e-5)), sd["out.2.weight"], sd["out.2.bias"], padding=1)
    return y.reshape(B, T, -1, H, W).permute(0, 2, 1, 3, 4)


def ddim_update_frames_f64(x, v_cond, v_uncond, noise, sc, frames, v_uncond_img=None, cfg_img=0.0):
    """float64 ops.ddim_update_frames: frame t of [B', C, T, H, W] takes frames[t]'s step scalars; the guidance combine and rescale
    (stds over the whole input) are sc's.  Returns fp64 (x_prev, pred_x0)."""
    d = lambda t: None if t is None else t.double()
    x, c, u, vi, nz = d(x), d(v_cond), d(v_uncond), d(v_uncond_img), d(noise)
    m = c
    if u is not None and sc["cfg_scale"] != 1.0:
        s = sc["cfg_scale"]
        m = u + s * (c - u) if vi is None else u + cfg_img * (vi - u) + s * (c - vi)
        g = sc["guidance_rescale"]
        if g > 0:
            m = g * (m * (c.std() / m.std())) + (1 - g) * m
    col = lambda key: torch.tensor([fr[key] for fr in frames], dtype=torch.float64, device=x.device).view(1, 1, -1, 1, 1)
    a_prev, sig = col("a_prev"), col("sigma_t")
    x0 = col("sqrt_ac_t") * x - col("sqrt_1mac_t") * m
    e_t = col("sqrt_ac_t") * m + col("sqrt_1mac_t") * x
    p0 = x0 * (col("prev_scale_t") / col("scale_t"))
    x_prev = a_prev.sqrt() * p0 + (1.0 - a_prev - sig * sig).clamp_min(0.0).sqrt() * e_t + sig * nz
    return x_prev, p0


def ddim_update_f64(x, v_cond, v_uncond, noise, sc, v_uncond_img=None, cfg_img=0.0):
    return dpm_update_f64(x, v_cond, v_uncond, noise, dict(sc, c_hist=0.0), torch.empty(x.shape, dtype=torch.float64, device=x.device),
                          v_uncond_img, cfg_img)


def fifo_loop(S, f, N, warm_start, denoise, draw, queue_coef):
    """The FIFO loop by its definition, one position at a time.
    warm_start() -> z [B, C, f, h, w];  draw(shape) -> the next random tensor;  queue_coef(k) -> (sqrt(a(tau_k)), sqrt(1 - a(tau_k)));
    denoise(p, x_window, renders, m) -> the window after one step (fp32), given the render index of every window position.
    Returns (out [B, C, N, h, w] fp32, log) with log = [(m, p, renders)] of every window evaluation."""
    z = warm_start()
    B, C, _, h, w = z.shape
    eps = draw((B, C, S, h, w))
    frames = []                                          # the queue as a list of S fp32 frames [B, C, h, w], head first
    for k in range(S):
        a, b = queue_coef(k)
        frames.append(a * z[:, :, max(0, k - (S - f))].float() + b * eps[:, :, k])
    out = [None] * N
    log = []
    for m in range(N + S - f):
        renders = [min(max(m + k - (S - f), 0), N - 1) for k in range(S)]
        new = list(frames)
        for p in range(S // f):
            pos = list(range(p * f, p * f + f))
            x = torch.stack([frames[k] for k in pos], 2)
            log.append((m, p, [renders[k] for k in pos]))
            y = denoise(p, x, [renders[k] for k in pos], m)
            for j, k in enumerate(pos):
                new[k] = y[:, :, j].float()
        frames = new
        if m - (S - f) >= 0:
            out[m - (S - f)] = frames[0]
        frames = frames[1:] + [draw((B, C, 1, h, w))[:, :, 0]]
    assert all(o is not None for o in out)
    return torch.stack(out, 2), log
