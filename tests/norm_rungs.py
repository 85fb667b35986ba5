"""The rung ladder of offset and degenerate activations and the float64 GroupNorm / LayerNorm reference shared by the statistics
tests (test_norm_statistics_gpu.py, test_peer_kernels_gpu.py).  See test_norm_statistics_gpu.py for the bounds."""
import math

import torch
import torch.nn.functional as F

# ------------------------------------------------------------------------------------------------ data ladder and reference
# name -> (eps, |mean| / std of a row or group as generated)
RUNGS = {
    "centred": (1e-5, 0.0),
    "mu16": (1e-5, 16.0),
    "mu64": (1e-5, 64.0),
    "mu256": (1e-5, 256.0),
    "chan50": (1e-5, 50.0),            # per-channel means over +-50, std 1 within a channel
    "big": (1e-5, 0.0),                # std 1e4
    "tiny-eps1e-5": (1e-5, 500.0),     # mean 0.5, std 1e-3: the variance sits below eps
    "tiny-eps1e-6": (1e-6, 500.0),
    "const-eps1e-5": (1e-5, math.inf),  # std 0
    "const-eps1e-6": (1e-6, math.inf),
}
RUNGS_EPS5 = [r for r in RUNGS if RUNGS[r][0] == 1e-5]      # for paths whose eps is fixed at 1e-5


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def rung_data(rung, rows, C, seed, samples=None):
    """fp16 [rows, C] on the rung.  const: one value per row, or per sample when `samples` is given (GroupNorm: every group of the
    sample, however the channels are grouped, is constant)."""
    g = _gen(seed)
    n = torch.randn(rows, C, generator=g, device="cuda")
    if rung == "centred":
        x = n
    elif rung.startswith("mu"):
        x = float(rung[2:]) + n
    elif rung == "chan50":
        x = (torch.rand(C, generator=g, device="cuda") * 100.0 - 50.0)[None, :] + n
    elif rung == "big":
        x = (n * 1e4).clamp(-6.0e4, 6.0e4)
    elif rung.startswith("tiny"):
        x = 0.5 + 1e-3 * n
    elif rung.startswith("const"):
        if samples is None:
            v = torch.randn(rows, 1, generator=g, device="cuda") * 100.0
            x = v.expand(rows, C)
        else:
            v = torch.randn(samples, 1, 1, generator=g, device="cuda") * 4.0
            x = v.expand(samples, rows // samples, C).reshape(rows, C)
    else:
        raise ValueError(rung)
    return x.to(torch.float16).contiguous()


def norm_ref(x, gamma, beta, eps, samples=None, groups=32, silu=False):
    """float64 LayerNorm over the last dim (samples=None) or GroupNorm(groups) of `samples` blocks of rows, from x as stored.
    Returns (y, mean, rstd): mean / rstd per row [rows], or per (sample, group) [samples, groups]."""
    xd = x.double()
    rows, C = xd.shape
    if samples is None:
        mean = xd.mean(1)
        var = (xd - mean[:, None]).square().mean(1)
        rstd = 1.0 / torch.sqrt(var + eps)
        xh = (xd - mean[:, None]) * rstd[:, None]
    else:
        v = xd.view(samples, rows // samples, groups, C // groups)
        mean = v.mean(dim=(1, 3))
        var = (v - mean[:, None, :, None]).square().mean(dim=(1, 3))
        rstd = 1.0 / torch.sqrt(var + eps)
        xh = ((v - mean[:, None, :, None]) * rstd[:, None, :, None]).view(rows, C)
    y = xh * gamma.double()[None, :] + beta.double()[None, :]
    if silu:
        y = F.silu(y)
    return y, mean, rstd


def affine(C, seed):
    g = _gen(seed)
    return (1.0 + 0.5 * torch.randn(C, generator=g, device="cuda")), 0.5 * torch.randn(C, generator=g, device="cuda")


# worst errors seen, (path, rung) -> {measure: value}; printed when the module ends
REPORT = {}


def _note(path, rung, **vals):
    d = REPORT.setdefault((path, rung), {})
    for k, v in vals.items():
        d[k] = max(d.get(k, 0.0), float(v))


def check_out(path, rung, y, ref, loose=None):
    """The output bound.  loose: (mask, extra) -- elements where `mask` holds get `extra` on top of the bound instead (see _gn_check)."""
    y = y.double()
    assert bool(torch.isfinite(y).all()), f"{path} {rung}: non-finite output"
    err = (y - ref).abs()
    bound = 3e-3 + 4e-3 * ref.abs()
    ratio = err / bound
    if loose is None:
        _note(path, rung, **{"out/bound": float(ratio.max())})
    else:
        mask, extra = loose
        if bool((~mask).any()):
            _note(path, rung, **{"out/bound": float(ratio[~mask].max())})
        if bool(mask.any()):
            _note(path, rung, **{"loose out/bound": float(ratio[mask].max())})
        bound = torch.where(mask, bound + extra, bound)
    bad = err > bound
    assert not bool(bad.any()), (f"{path} {rung}: max err {float(err.max()):.4g} (ref absmax {float(ref.abs().max()):.4g}), "
                                 f"{int(bad.sum())} / {bad.numel()} outside the bound")


def check_stats(path, rung, mean, rstd, mean_ref, rstd_ref, eps):
    mean, rstd = mean.double(), rstd.double()
    rel = ((rstd - rstd_ref) / rstd_ref).abs()
    dm = (mean - mean_ref).abs() * rstd_ref
    _note(path, rung, rstd_rel=float(rel.max()), **{"mean*rstd": float(dm.max())})
    assert float(rel.max()) <= 2e-4, f"{path} {rung}: rstd relative error {float(rel.max()):.3g}"
    assert float(dm.max()) <= 2e-4, f"{path} {rung}: |mean error| * rstd = {float(dm.max()):.3g}"
    if rung.startswith("const"):
        worst = float(((rstd - eps ** -0.5) / eps ** -0.5).abs().max())
        assert worst <= 1e-6, f"{path} {rung}: constant rows give rstd off eps^-0.5 by {worst:.3g}"


GN_STRICT_SHIFT = 64.0


def _gn_check(path, rung, out, x, samples, gamma, beta, eps, silu):
    """GroupNorm output against norm_ref.  Groups with |mean| / std <= GN_STRICT_SHIFT get the output bound.  The others (constant groups
    included) get a regression bound: an rstd error of 5 % and a mean error of 5 % of the std, i.e. 0.06 |gamma| (|xhat| + 1), plus the
    fp32 rounding of the normalise pass's shift beta - mean * rstd * gamma, 1e-6 |gamma mean rstd|."""
    ref, mean, rstd = norm_ref(x, gamma, beta, eps, samples=samples, silu=silu)
    xh, _, _ = norm_ref(x, torch.ones_like(gamma), torch.zeros_like(gamma), eps, samples=samples)
    rows, C = x.shape
    std = x.double().view(samples, rows // samples, 32, C // 32).std(dim=(1, 3), unbiased=False)
    wide = mean.abs() > GN_STRICT_SHIFT * std                                   # [samples, 32]; std == 0: any non-zero mean
    per_elem = lambda t: t[:, None, :, None].expand(samples, rows // samples, 32, C // 32).reshape(rows, C)
    ga = gamma.double().abs()[None, :]
    extra = 0.06 * ga * (xh.abs() + 1.0) + 1e-6 * ga * per_elem(mean.abs() * rstd)
    check_out(path, rung, out, ref, loose=(per_elem(wide), extra))
