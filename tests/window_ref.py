"""Independent restatements of windowed temporal attention (FreeNoise) for the tests: the window definition, a float64 reference of
`ops.temporal_attn_windowed` with its error bound, the noise rescheduling, and the fp32 oracle U-Net with windowed temporal attention.

The bound: out_t = sum_win w O_win(t) / sum_win w is a convex combination of the windows' attention outputs, so blending the
per-window bounds of `attention_ref.attn_bound` with the same weights bounds |out_t - ref_t| up to the fp32 blend (a few 2^-24
relative, far below the fp16 store's u that the per-window bound already carries once)."""
from __future__ import annotations

import contextlib

import torch

from tests import attention_ref as ar


def starts(T, W, S):
    """Window starts by the definition: 0, S, 2S, ... while start + W < T, plus T - W if not yet listed."""
    out = []
    s = 0
    while s + W < T:
        out.append(s)
        s += S
    if T - W not in out:
        out.append(max(T - W, 0))
    return out


def weights(W):
    return [min(j + 1, W - j) for j in range(W)]


def weight_sums(T, W, S):
    """Per-frame sum of the blend weights, by brute force over the windows."""
    tot = [0] * T
    for s in starts(T, W, S):
        for j, w in enumerate(weights(min(W, T))):
            tot[s + j] += w
    return tot


def reschedule(x, W, S, seed):
    """FreeNoise's rescheduling by its definition, one frame at a time on a list of frames."""
    g = torch.Generator().manual_seed(seed)
    frames = [x[:, :, t].clone() for t in range(x.shape[2])]
    i = W
    while i < len(frames):
        perm = torch.randperm(S, generator=g).tolist()
        for j in range(min(S, len(frames) - i)):
            frames[i + j] = frames[i - W + perm[j]].clone()
        i += S
    return torch.stack(frames, 2)


def windowed_ref(q, k, v, W, S, scale=0.125):
    """float64 windowed attention and its bound over [..., T, 64] tensors (T on dim -2)."""
    T = q.shape[-2]
    if T <= W:
        o, p, mag = ar.attn_ref(q, k, v, scale)
        return o, ar.attn_bound(o, p, mag, v)
    out = torch.zeros(q.shape, dtype=torch.float64, device=q.device)
    bnd = torch.zeros_like(out)
    tot = torch.zeros(T, dtype=torch.float64, device=q.device)
    w = torch.tensor(weights(W), dtype=torch.float64, device=q.device)[:, None]
    for s in starts(T, W, S):
        sl = slice(s, s + W)
        o, p, mag = ar.attn_ref(q[..., sl, :], k[..., sl, :], v[..., sl, :], scale)
        out[..., sl, :] += w * o
        bnd[..., sl, :] += w * ar.attn_bound(o, p, mag, v[..., sl, :])
        tot[sl] += w[:, 0]
    return out / tot[:, None], bnd / tot[:, None]


@contextlib.contextmanager
def oracle_window(window):
    """Inside the block, the fp32 oracle (oracle.lvdm_oracle) runs every temporal transformer's self-attentions on windows (W, S)
    blended by the definition; spatial and cross-attention are untouched.  None: the oracle as it is."""
    from oracle import lvdm_oracle as O
    if window is None:
        yield
        return
    W, S = window
    tt, attend = O.temporal_transformer, O._attend

    def windowed_attend(q, k, v, scale):                       # q, k, v: [b, h, T, d], T = frames
        T = q.shape[2]
        if T <= W:
            return attend(q, k, v, scale)
        out = torch.zeros_like(q)
        tot = torch.zeros(T, dtype=q.dtype)
        wt = torch.tensor(weights(W), dtype=q.dtype)[:, None]
        for s in starts(T, W, S):
            sl = slice(s, s + W)
            out[:, :, sl] += wt * attend(q[:, :, sl], k[:, :, sl], v[:, :, sl], scale)
            tot[sl] += wt[:, 0]
        return out / tot[:, None]

    def temporal_transformer(sd, p, x, T):
        O._attend = windowed_attend
        try:
            return tt(sd, p, x, T)
        finally:
            O._attend = attend

    O.temporal_transformer = temporal_transformer
    try:
        yield
    finally:
        O.temporal_transformer = tt
