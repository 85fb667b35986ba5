"""Inputs, float64 references and a derived error bound for the attention kernels (`flash_attn`, `temporal_attn`, `softmax_rows`).

Rungs.  Centred Gaussian q and k give logits of standard deviation 1 or less, on which a softmax that never subtracts its running max,
or lets one padded key in, still lands within a few 1e-3 of the truth.  Each rung sets the logit distribution directly instead:

    centred, peaked4, peaked16     logit std 1, 4, 16 (16: nearly one-hot rows)
    shift+30, shift-30             every logit ~ +-30 + N(0,1): a missing max subtraction overflows fp16 at +30; a key that was
                                   zero-filled by TMA (logit exactly 0) would own the row at -30
    late-max@j                     key j sits 20 above the N(0,1) rest: the whole history is rescaled when its tile arrives
                                   (j = last, lasttile = the first key of the last tile, 63, 64, 127, 128)
    sink10, sink15                 key 0 sits 10 / 15 above the bulk: at 9216 keys the bulk probabilities are fp16 subnormals
    ramp                           the logit rises by 16 over the key axis, so the running max rises in every tile
    ties                           all keys identical: the answer is mean(V)
    v-offset, v-large              centred logits with V = 50 + N(0,1) (catches a leaked key and any l / sum(P) mismatch),
                                   or V of std 1e3

The bias rungs use head dimension 0: q[:, 0] = 16 and k[:, 0] = b so that the logit gets 0.125 * 16 * b on top of an N(0,1) bulk
carried by dimensions 1..63.

Bound.  For output element (query i, column c) of softmax(s) V with s = scale * q k^T (u = 2^-11, the fp16 unit roundoff):

    bound = C1 * u * (|o_ic| + sum_j p_ij |v_jc|)                  (a)
          + sum_j p_ij |v_jc - o_ic| * ds_ij                       (b)
          + Nk * 2^-25 * max_j |v_jc|                              (c)
          + 2^-24                                                  (d)
          [+ u * |base_ic + o_ic|]                                 (e)  accumulate=True only

(a) The kernels round the unnormalised probabilities e = exp(s - m) in (0, 1] to fp16 for the P V product (relative u on normal
values) while l sums the unrounded e in fp32, and they round O / l to fp16 once (relative u).  That is 1 * u on each sum.  The fp32
arithmetic adds, at most: l's per-thread running sum over Nk / 4 keys (Nk/4 * 2^-24), the P V accumulator's chain of Nk/16 wgmma k-steps
plus one alpha rescale per tile (< Nk/16 + Nk/64 roundings of 2^-23, truncating accumulation assumed) and ex2.approx (2^-22).  Below
Nk = 20165 those sum to less than one more u, so C1 = 2; `attn_bound` refuses longer rows.  The running-max rescale factor alpha
multiplies O and l alike and cancels.
(b) A logit error ds_ij moves o_i by sum_j p_ij ds_ij (v_j - o_i) to first order.  ds_ij = GAMMA_S * scale * sum_k |q_ik k_jk|: the
64-term fp32 dot product (64 * 2^-23, truncating accumulation) and the fp32 rounding of s * scale * log2(e) - m (2^-23 |s| <=
2^-23 scale sum_k |q k|), so GAMMA_S = 65 * 2^-23.  |v_jc - o_ic| is bounded by |v_jc - mean_j v_jc| + |o_ic - mean_j v_jc|.
(c) e below 2^-14 rounds to an fp16 subnormal with an absolute error of at most 2^-25, and l >= 1 (the key at the running max has
e = 1).
(d) the output's own subnormal floor; (e) the second rounding of the accumulate epilogue.

`softmax_bound` is the bound for `softmax_rows`; its derivation is in its docstring.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -11
C1 = 2.0
GAMMA_S = 65 * 2.0 ** -23
MAX_NK = 16384

RUNGS = ["centred", "peaked4", "peaked16", "shift+30", "shift-30", "late-max@last", "late-max@lasttile", "late-max@63", "late-max@64",
         "late-max@127", "late-max@128", "sink10", "sink15", "ramp", "ties", "v-offset", "v-large"]

BIAS_Q = 16.0          # q[:, 0] on the bias rungs


def late_max_key(rung: str, Nk: int, bnk: int = 64):
    """Index of the raised key of a late-max rung, or None when the rung does not exist for Nk keys."""
    at = rung.split("@")[1]
    j = Nk - 1 if at == "last" else (Nk - 1) // bnk * bnk if at == "lasttile" else int(at)
    return j if j < Nk else None


def rungs_for(Nk: int, bnk: int = 64):
    """The rungs that exist for Nk keys: late-max@j needs j < Nk, and lasttile only differs from a fixed j past one tile."""
    out = []
    for r in RUNGS:
        if r.startswith("late-max@"):
            j = late_max_key(r, Nk, bnk)
            if j is None or (r == "late-max@lasttile" and Nk <= bnk):
                continue
        out.append(r)
    return out


def _bulk(shape, logit_std, dims, scale, g, device):
    """N(0, a^2) entries whose `dims`-term dot products times `scale` have standard deviation `logit_std`."""
    a = math.sqrt(logit_std / (scale * math.sqrt(dims)))
    return torch.randn(*shape, generator=g, device=device) * a


def rung_qkv(rung: str, G: int, Nq: int, Nk: int, heads: int, seed: int, device="cuda", scale: float = 0.125, Gk: int = None,
             bnk: int = 64):
    """fp16 q [G, Nq, heads, 64], k and v [Gk, Nk, heads, 64] (Gk defaults to G) whose logits scale * q . k follow the rung."""
    Gk = G if Gk is None else Gk
    g = torch.Generator(device=device).manual_seed(seed)
    qs, ks = (G, Nq, heads, 64), (Gk, Nk, heads, 64)
    v = torch.randn(*ks, generator=g, device=device)
    if rung == "v-offset":
        v = v + 50.0
    elif rung == "v-large":
        v = v * 1e3
    if rung in ("centred", "peaked4", "peaked16", "v-offset", "v-large", "ties"):
        std = {"peaked4": 4.0, "peaked16": 16.0}.get(rung, 1.0)
        q, k = _bulk(qs, std, 64, scale, g, device), _bulk(ks, std, 64, scale, g, device)
        if rung == "ties":
            k = k[:, :1].expand(ks).contiguous()
        return q.half(), k.half(), v.half()
    q = _bulk(qs, 1.0, 63, scale, g, device)
    k = _bulk(ks, 1.0, 63, scale, g, device)
    q[..., 0] = BIAS_Q
    per = 1.0 / (scale * BIAS_Q)           # k[:, 0] per nat of logit
    if rung in ("shift+30", "shift-30"):
        k[..., 0] = (30.0 if rung == "shift+30" else -30.0) * per
    elif rung.startswith("late-max@"):
        k[..., 0] = 0.0
        k[:, late_max_key(rung, Nk, bnk), :, 0] = 20.0 * per
    elif rung.startswith("sink"):
        k[..., 0] = 0.0
        k[:, 0, :, 0] = float(rung[4:]) * per
    elif rung == "ramp":
        k[..., 0] = (16.0 * per / max(Nk - 1, 1)) * torch.arange(Nk, device=device, dtype=torch.float32)[None, :, None]
    else:
        raise ValueError(rung)
    return q.half(), k.half(), v.half()


def attn_ref(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float):
    """float64 softmax(scale q k^T) v over the last two dims of the tensors as stored ([..., N, 64]).
    Returns o [..., Nq, 64], p [..., Nq, Nk] and mag = scale * |q| |k|^T [..., Nq, Nk], the magnitude the logit error scales with."""
    qd, kd, vd = q.double(), k.double(), v.double()
    s = scale * (qd @ kd.transpose(-1, -2))
    p = torch.softmax(s, -1)
    return p @ vd, p, scale * (qd.abs() @ kd.abs().transpose(-1, -2))


def attn_bound(o: torch.Tensor, p: torch.Tensor, mag: torch.Tensor, v: torch.Tensor, base: torch.Tensor = None) -> torch.Tensor:
    """The bound of the module docstring for each element of o ([..., Nq, 64]); v as stored, base: the accumulate target."""
    Nk = v.shape[-2]
    assert Nk <= MAX_NK, f"C1 = {C1} is derived for at most {MAX_NK} keys"
    vd = v.double()
    av = vd.abs()
    mu = vd.mean(-2, keepdim=True)
    w = p * (GAMMA_S * mag)
    b = C1 * U * (o.abs() + p @ av)
    b = b + w @ (vd - mu).abs() + (o - mu).abs() * w.sum(-1, keepdim=True)
    b = b + Nk * 2.0 ** -25 * av.amax(-2, keepdim=True) + 2.0 ** -24
    if base is not None:
        b = b + U * (base.double() + o).abs()
    return b


def softmax_ref(scores: torch.Tensor, scale: float) -> torch.Tensor:
    """float64 row softmax of scale * scores (-inf entries get probability 0)."""
    return torch.softmax(scores.double() * scale, -1)


def softmax_bound(scores: torch.Tensor, scale: float) -> torch.Tensor:
    """Bound on |p - ref| for `softmax_rows`, which computes e_j = __expf((x_j - m) * scale), l = sum e_j in fp32 (per thread over
    ceil(cols / 256) columns, then a 5-level warp tree, then 8 warps in order), and p_j = fp16(e_j * (1 / l)).

    - a_j = (x_j - m) * scale is rounded twice: its error is 2^-23 |a_j| in the exponent, a relative error of 2^-23 |a_j| in e_j.
    - __expf(a) is accurate to 2 + floor(1.173 |a|) ulp (CUDA C Programming Guide, intrinsic functions): (2 + 1.173 |a_j|) 2^-23.
    - l carries the weighted mean of those, sum_j p_j eps_j, plus (ceil(cols / 256) + 13) 2^-24 from its summation.
    - 1 / l and e * inv round once each: 2 * 2^-24.
    - the fp16 store: u p on normal values, 2^-25 below 2^-14.
    So |p_j - ref_j| <= u ref_j + 2^-25 + ref_j (eps_j + eps_l + 2^-23), with eps_j = (2 + 2.173 |a_j|) 2^-23, times (1 + 2^-10) for the
    second-order products."""
    x = scores.double()
    ref = softmax_ref(scores, scale)
    m = x.amax(-1, keepdim=True)
    a = ((x - m) * scale).abs()
    eps = torch.where(ref > 0, (2.0 + 2.173 * a) * 2.0 ** -23, torch.zeros_like(a))
    depth = math.ceil(x.shape[-1] / 256) + 13
    eps_l = (ref * eps).sum(-1, keepdim=True) + depth * 2.0 ** -24
    return (U * ref + 2.0 ** -25 + ref * (eps + eps_l + 2.0 ** -23)) * (1 + 2.0 ** -10)


def worst_ratio(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |out - ref| / bound; inf when out has a non-finite element."""
    out = out.double()
    if not bool(torch.isfinite(out).all()):
        return math.inf
    return float(((out - ref).abs() / bound).max())
