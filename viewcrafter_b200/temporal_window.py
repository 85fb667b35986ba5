"""Windowed temporal attention and noise rescheduling for clips longer than the checkpoints' 16 / 25 frames: FreeNoise (Qiu et al.,
ICLR 2024), built on VideoCrafter's lvdm 3-D U-Net, which this library implements (INTEGRATION.md "Long clips: windowed temporal
attention").

A window is (W, S): every temporal self-attention runs on windows of W frames at starts 0, S, 2S, ... (while start + W < T) plus a
last one at T - W, and frame t's output is the mean of the windows' outputs for t weighted by min(j + 1, W - j), j = t - start.
The kernel (`ops.temporal_attn_windowed`) computes the weight sums with `weight_sum`'s arithmetic; `window_starts` and
`weight_sum` state that arithmetic on the host.  `reschedule_noise` is the second half of FreeNoise, applied to x_T by the samplers.
"""
from __future__ import annotations

import operator
from typing import List, Optional, Tuple

import torch

MAX_W = 32          # one warp's 32 x 32 score tile


def check_window(window) -> Optional[Tuple[int, int]]:
    """None (off), or (W, S) with 2 <= W <= 32 and 1 <= S <= W, returned as a tuple of ints.  Anything else raises ValueError."""
    if window is None:
        return None
    try:
        W, S = window
        if isinstance(W, bool) or isinstance(S, bool):
            raise TypeError
        W, S = operator.index(W), operator.index(S)
    except (TypeError, ValueError):
        raise ValueError(f"temporal window must be None or a pair of ints (W, S), got {window!r}") from None
    if not (2 <= W <= MAX_W and 1 <= S <= W):
        raise ValueError(f"temporal window (W, S) = ({W}, {S}) out of range: 2 <= W <= {MAX_W} and 1 <= S <= W")
    return W, S


def window_starts(T: int, W: int, S: int) -> List[int]:
    """Starts of the windows over T frames: 0, S, 2S, ... while start + W < T, then T - W; [0] when T <= W."""
    if T <= W:
        return [0]
    return list(range(0, T - W, S)) + [T - W]


def weight_sum(t: int, T: int, W: int, S: int) -> int:
    """Sum of the blend weights min(j + 1, W - j) of the windows that contain frame t (T > W), from (t, T, W, S) alone, as the kernel
    computes it: the regular windows i * S with t - W < i * S <= t, plus the last window T - W when it contains t."""
    n = (T - W + S - 1) // S + 1
    total = 0
    i = 0 if t < W else (t - W) // S + 1
    while i < n - 1 and i * S <= t:
        j = t - i * S
        total += min(j + 1, W - j)
        i += 1
    if t >= T - W:
        total += min(t - (T - W) + 1, T - t)
    return total


def reschedule_noise(x: torch.Tensor, window, seed: int = 0) -> torch.Tensor:
    """FreeNoise's noise rescheduling of an initial latent x [B, C, T, h, w] (returns a new tensor; x is not modified).  For
    i = W, W + S, W + 2S, ... < T in order, frames i .. min(i + S, T) - 1 take the (already rescheduled) noise of frames
    (i - W) + perm[:len], where perm = torch.randperm(S) from a CPU generator seeded with `seed` and created here, one
    permutation per chunk.  Every batch row gets the same permutation, so row b of a rescheduled batch is row b rescheduled alone.
    The global CPU and device generators are not touched."""
    W, S = check_window(window)
    T = x.shape[2]
    g = torch.Generator().manual_seed(int(seed))
    y = x.clone()
    for i in range(W, T, S):
        n = min(i + S, T) - i
        src = (i - W) + torch.randperm(S, generator=g)[:n]
        y[:, :, i:i + n] = y[:, :, src.to(y.device)]
    return y
