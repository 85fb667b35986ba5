"""The attention kernels on peaked, shifted and tile-edge softmax inputs against float64, inside a derived fp16 error bound.

Paths: `flash_attn` (both tile widths: chosen by key count in this process, and each forced for every shape in a child process, because
the choice is cached per process), the U-Net's exact call sequences at level 0, the resampler's call, `temporal_attn` (every T, sites
that are not a multiple of 4 warps, and the level-0 grid that strides), `softmax_rows` and the VAE AttnBlock end to end.  Inputs are the
rungs of `tests/attention_ref.py`; every result is compared with a float64 reference of the fp16 tensors as stored, through the bound
derived there.  The worst |out - ref| / bound per path and rung is printed when the module ends: run with ``-s`` to see the table.

Run as ``python tests/test_attention_numerics_gpu.py --bn64 {0,1}``, the module checks the forced-width case list on one tile width,
prints its table and ATTN_NUMERICS_OK (what `test_forced_tile_width` does).
"""
import argparse
import math
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import pytest
import torch

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import attention_ref as ar

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

SENTINEL = "ATTN_NUMERICS_OK"
CHUNK = 1 << 24            # fp64 elements per [rows, keys] reference block


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


# worst |out - ref| / bound, (path, rung) -> value; printed when the module ends
REPORT = {}
_T0 = time.time()


def _note(path, rung, r):
    REPORT[(path, rung)] = max(REPORT.get((path, rung), 0.0), r)


def _table(report):
    lines = [f"{'path':28s} {'rung':18s} {'worst |out-ref|/bound':>22s}"]
    lines += [f"{p:28s} {r:18s} {v:22.3g}" for (p, r), v in sorted(report.items())]
    return "\n".join(lines)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print(f"\nattention numerics: worst |out - ref| / bound per path and rung ({time.time() - _T0:.0f} s)\n" + _table(REPORT))


def _check(path, rung, r, what):
    _note(path, rung, r)
    assert r <= 1.0, f"{path} {rung} {what}: |out - ref| / bound = {r:.4g}"


def _tile_keys(Nk):
    """Key-tile width flash_attn runs for Nk keys in this process (VC_ATTN_BN64 forces it)."""
    mode = os.environ.get("VC_ATTN_BN64")
    if mode is not None:
        return 64 if mode.startswith("1") else 128
    return 64 if Nk <= 1024 else 128


def _ratio_heads(out, q, k, v, base=None, extra=None):
    """Worst ratio of out [..., Nq, 64] against attention over q [..., Nq, 64], k / v [..., Nk, 64] (+ base), in query chunks.
    extra: (k2, v2): out is attention over (k, v) accumulated with attention over (k2, v2), as the U-Net's image path does."""
    Nq, Nk = q.shape[-2], k.shape[-2]
    pairs = q.numel() // (Nq * 64)
    step = max(1, CHUNK // (pairs * Nk * (2 if extra is None else 4)))
    worst = 0.0
    for r0 in range(0, Nq, step):
        rs = (..., slice(r0, r0 + step), slice(None))
        o, p, mag = ar.attn_ref(q[rs], k, v, 0.125)
        b = None if base is None else base[rs]
        bound = ar.attn_bound(o, p, mag, v, base=b)
        ref = o if b is None else o + b.double()
        if extra is not None:
            o2, p2, mag2 = ar.attn_ref(q[rs], *extra, 0.125)
            bound = bound + ar.attn_bound(o2, p2, mag2, extra[1], base=ref)
            ref = ref + o2
        worst = max(worst, ar.worst_ratio(out[rs], ref, bound))
    return worst


def _pairs(B, heads, Nq, Nk):
    """(b, [heads]) to compare: all of them on small problems, the corners and the middle on large ones."""
    if B * heads * Nq * Nk <= 1 << 24:
        return [(b, list(range(heads))) for b in range(B)]
    hs = sorted({0, heads // 2, heads - 1})
    return sorted({(0, tuple(hs)), (B - 1, tuple(hs))})


def flash_case(ops, rung, B, heads, Nq, Nk, shared=False, accumulate=False, seed=0):
    """q, k and v as column views of one [rows, 3C] tensor; returns the worst ratio over the compared (batch, head) pairs."""
    C = heads * 64
    Gk = 1 if shared else B
    q, k, v = ar.rung_qkv(rung, B, Nq, Nk, heads, seed, Gk=Gk, bnk=_tile_keys(Nk))
    qkv = torch.zeros((max(B * Nq, Gk * Nk), 3 * C), device="cuda", dtype=torch.float16)
    qkv[:B * Nq, :C] = q.reshape(B * Nq, C)
    qkv[:Gk * Nk, C:2 * C] = k.reshape(Gk * Nk, C)
    qkv[:Gk * Nk, 2 * C:] = v.reshape(Gk * Nk, C)
    base = None
    if accumulate:
        base = (torch.randn(B * Nq, C, generator=torch.Generator(device="cuda").manual_seed(seed + 7), device="cuda") * 4.0).half()
    out = ops.flash_attn(qkv[:B * Nq, :C], qkv[:Gk * Nk, C:2 * C], qkv[:Gk * Nk, 2 * C:], B, Nq, Nk, heads, kv_shared=shared,
                         out=None if base is None else base.clone(), accumulate=accumulate)
    assert bool(torch.isfinite(out).all()), "non-finite output"
    out4 = out.view(B, Nq, heads, 64)
    base4 = None if base is None else base.view(B, Nq, heads, 64)
    worst = 0.0
    for b, hs in _pairs(B, heads, Nq, Nk):
        hs = list(hs)
        bk = 0 if shared else b
        sel = lambda t, i: t[i][:, hs].transpose(0, 1)
        worst = max(worst, _ratio_heads(sel(out4, b), sel(q, b), sel(k, bk), sel(v, bk),
                                        base=None if base4 is None else sel(base4, b)))
    return worst


# ------------------------------------------------------------------------------------------------ flash_attn, tile width by key count
# (B, heads, Nq, Nk, kv_shared, accumulate): every Nk edge of both tile widths and the 1024 / 1025 switch, Nq from one row to a partial
# last CTA (Nq <= 64 leaves the second MMA warpgroup without rows)
FLASH_CASES = [
    (2, 1, 1, 1, False, False), (2, 5, 16, 16, False, False), (2, 10, 64, 63, False, False), (2, 20, 65, 64, False, False),
    (2, 1, 128, 65, True, False), (2, 5, 129, 77, True, True), (2, 10, 576, 127, False, False), (2, 20, 1, 128, False, False),
    (2, 1, 16, 129, False, True), (2, 5, 64, 256, True, False), (2, 10, 65, 1000, False, False), (2, 20, 128, 1024, False, False),
    (2, 1, 129, 1025, False, False), (2, 5, 576, 2304, False, False), (1, 10, 64, 9216, False, False), (1, 5, 576, 9216, True, False),
    (2, 20, 129, 1025, False, True),
]
FLASH_PARAMS = [(c, r) for c in FLASH_CASES for r in ar.rungs_for(c[3], _tile_keys(c[3]))]


@pytest.mark.parametrize("case,rung", FLASH_PARAMS, ids=[f"{'-'.join(map(str, c[:4]))}{'-sh' if c[4] else ''}{'-acc' if c[5] else ''}-{r}"
                                                          for c, r in FLASH_PARAMS])
def test_flash_attn(ops, case, rung):
    B, heads, Nq, Nk, shared, acc = case
    _check("flash auto" + (" acc" if acc else ""), rung, flash_case(ops, rung, B, heads, Nq, Nk, shared, acc), str(case))


# ------------------------------------------------------------------------------------------------ the U-Net's and resampler's calls
T0, HW0, HEADS0 = 25, 9216, 5           # level 0 of the 576x1024x25 forward
SEQ_RUNGS = ["centred", "peaked16", "shift-30", "shift+30", "late-max@last", "sink15", "v-offset"]


@pytest.mark.parametrize("rung", SEQ_RUNGS)
def test_unet_self_attention(ops, rung):
    """_spatial_tf attn1: q / k / v column views of the [T*HW, 3C] qkv GEMM output, B = T frames of HW tokens."""
    C = HEADS0 * 64
    q, k, v = ar.rung_qkv(rung, T0, HW0, HW0, HEADS0, 11, bnk=_tile_keys(HW0))
    qkv = torch.cat([t.reshape(T0 * HW0, C) for t in (q, k, v)], 1)
    out = ops.flash_attn(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], T0, HW0, HW0, HEADS0).view(T0, HW0, HEADS0, 64)
    assert bool(torch.isfinite(out).all())
    worst = 0.0
    for t, h in ((0, 0), (T0 // 2, 2), (T0 - 1, HEADS0 - 1)):
        worst = max(worst, _ratio_heads(out[t, :, h][None], q[t, :, h][None], k[t, :, h][None], v[t, :, h][None]))
    _check("unet self", rung, worst, "")


@pytest.mark.parametrize("image", ["per-frame", "shared256"])
@pytest.mark.parametrize("rung", SEQ_RUNGS)
def test_unet_cross_attention_sequence(ops, rung, image):
    """_spatial_tf attn2 for batch element b = 1: text attention over 77 shared keys into a[rows], then the image attention accumulated
    into the same rows -- per frame (16 keys per frame, K / V batched by frame) or over 256 shared keys."""
    C, T, HW = HEADS0 * 64, T0, HW0
    q, kt, vt = ar.rung_qkv(rung, T, HW, 77, HEADS0, 21, Gk=1)
    nki, Gi = (16, T) if image == "per-frame" else (256, 1)
    _, ki, vi = ar.rung_qkv(rung, T, HW, nki, HEADS0, 22, Gk=Gi)
    qall = torch.randn(2 * T * HW, C, device="cuda").half()
    rows = slice(T * HW, 2 * T * HW)
    qall[rows] = q.reshape(T * HW, C)
    kv_txt = torch.cat([kt.reshape(77, C), vt.reshape(77, C)], 1)
    kv_img = torch.cat([ki.reshape(Gi * nki, C), vi.reshape(Gi * nki, C)], 1)
    a = torch.empty_like(qall)
    ops.flash_attn(qall[rows], kv_txt[:, :C], kv_txt[:, C:], T, HW, 77, HEADS0, kv_shared=True, out=a[rows])
    if image == "per-frame":
        ops.flash_attn(qall[rows], kv_img[:, :C], kv_img[:, C:], T, HW, kv_img.shape[0] // T, HEADS0, out=a[rows], accumulate=True)
    else:
        ops.flash_attn(qall[rows], kv_img[:, :C], kv_img[:, C:], T, HW, kv_img.shape[0], HEADS0, kv_shared=True, out=a[rows],
                       accumulate=True)
    out = a[rows].view(T, HW, HEADS0, 64)
    assert bool(torch.isfinite(out).all())
    worst = 0.0
    for t in (0, T // 2, T - 1):
        ti = t if image == "per-frame" else 0
        sel = lambda x, i: x[i].transpose(0, 1)
        worst = max(worst, _ratio_heads(sel(out, t), sel(q, t), sel(kt, 0), sel(vt, 0), extra=(sel(ki, ti), sel(vi, ti))))
    _check(f"unet text+{image}", rung, worst, "")


@pytest.mark.parametrize("rung", ar.rungs_for(257 + 256))
def test_resampler_attention(ops, rung):
    """resampler.py PerceiverAttention: L = 256 latent queries over 257 image tokens + the latents, 16 heads, q from its own GEMM and
    k / v column views of the [B*nk, 2*inner] kv GEMM output."""
    B, L, heads = 2, 256, 16
    nk, inner = 257 + L, heads * 64
    q, k, v = ar.rung_qkv(rung, B, L, nk, heads, 31, bnk=_tile_keys(nk))
    kv = torch.cat([k.reshape(B * nk, inner), v.reshape(B * nk, inner)], 1)
    out = ops.flash_attn(q.reshape(B * L, inner).contiguous(), kv[:, :inner], kv[:, inner:], B, L, nk, heads, scale=0.125)
    out = out.view(B, L, heads, 64)
    assert bool(torch.isfinite(out).all())
    worst = max(_ratio_heads(out[b].transpose(0, 1), q[b].transpose(0, 1), k[b].transpose(0, 1), v[b].transpose(0, 1)) for b in range(B))
    _check("resampler", rung, worst, "")


# ------------------------------------------------------------------------------------------------ flash_attn, tile width forced
# every case the previous per-width check ran, (B, heads, Nq, Nk, kv_shared, accumulate), then the tile edges of both widths
FORCED_CASES = [
    (2, 2, 256, 128, False, False), (1, 3, 300, 300, False, False), (2, 2, 130, 77, True, False), (1, 2, 384, 256, True, True),
    (2, 5, 640, 1000, False, False), (1, 5, 2304, 2304, False, False), (1, 2, 1024, 9216, True, False),
    (1, 1, 65, 1, False, False), (2, 1, 129, 63, False, False), (1, 2, 64, 65, False, True), (2, 1, 128, 127, False, False),
    (1, 1, 16, 129, True, False), (1, 2, 576, 1025, False, True), (1, 5, 129, 1024, True, False),
]
FORCED_RUNGS = ["centred", "peaked16", "shift-30", "shift+30", "late-max@last", "v-offset"]


def _forced_main(bn64):
    os.environ["VC_ATTN_BN64"] = str(bn64)
    from viewcrafter_b200 import ops as _ops
    path = f"flash bn{64 if bn64 else 128} forced"
    failed = []
    for case in FORCED_CASES:
        for rung in FORCED_RUNGS:
            r = flash_case(_ops, rung, *case)
            p = path + (" acc" if case[5] else "")
            _note(p, rung, r)
            print(f"RATIO\t{p}\t{rung}\t{r!r}\t{case}")
            if not r <= 1.0:
                failed.append((case, rung, r))
    print(_table(REPORT))
    for f in failed:
        print("FAILED", f)
    if not failed:
        print(SENTINEL)
    return 1 if failed else 0


@pytest.mark.parametrize("bn64", [0, 1])
def test_forced_tile_width(ops, bn64):
    """Each tile width for every shape of FORCED_CASES, in a fresh process (the width is chosen once per process)."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--bn64", str(bn64)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=540, env=dict(os.environ, VC_ATTN_BN64=str(bn64)))
    for line in r.stdout.splitlines():
        if line.startswith("RATIO\t"):
            _, path, rung, val, _case = line.split("\t")
            _note(path, rung, float(val))
    assert r.returncode == 0 and SENTINEL in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]


# ------------------------------------------------------------------------------------------------ temporal_attn
TEMPORAL_RUNGS = ar.rungs_for(T0)


def temporal_case(ops, rung, B, T, sites, heads, seed=0):
    """temporal_attn per batch element on the `rows` slices of a [B*T*sites, 3C] qkv (ld = 3C), rows at (t * sites + site)."""
    C = heads * 64
    q, k, v = ar.rung_qkv(rung, B * sites, T, T, heads, seed)                    # [B*sites, T, heads, 64]
    rows_of = lambda t: t.view(B, sites, T, C).transpose(1, 2).reshape(B * T * sites, C)
    qkv = torch.cat([rows_of(q), rows_of(k), rows_of(v)], 1)
    a = torch.empty((B * T * sites, C), device="cuda", dtype=torch.float16)
    for b in range(B):
        rows = slice(b * T * sites, (b + 1) * T * sites)
        ops.temporal_attn(qkv[rows, :C], qkv[rows, C:2 * C], qkv[rows, 2 * C:], T, sites, heads, out=a[rows])
    assert bool(torch.isfinite(a).all())
    out = a.view(B, T, sites, heads, 64).permute(0, 2, 3, 1, 4).reshape(B * sites, heads, T, 64)
    per = lambda t: t.transpose(1, 2)                                             # [B*sites, heads, T, 64]
    worst, step = 0.0, max(1, CHUNK // (heads * T * T * 8))
    for g0 in range(0, B * sites, step):
        gs = slice(g0, g0 + step)
        worst = max(worst, _ratio_heads(out[gs], per(q[gs]), per(k[gs]), per(v[gs])))
    return worst


@pytest.mark.parametrize("rung", ["centred", "peaked16"])
@pytest.mark.parametrize("T", list(range(1, 33)))
def test_temporal_attn_every_T(ops, T, rung):
    _check("temporal T sweep", rung, temporal_case(ops, rung, 1, T, 33, 2, seed=T), f"T={T}")


@pytest.mark.parametrize("rung", TEMPORAL_RUNGS)
def test_temporal_attn_rungs(ops, rung):
    _check("temporal T25", rung, temporal_case(ops, rung, 2, T0, 144, 5, seed=41), "sites=144")


@pytest.mark.parametrize("rung", ["centred", "shift-30", "late-max@last"])
@pytest.mark.parametrize("sites", [7, 33])
def test_temporal_attn_odd_sites(ops, sites, rung):
    """sites * heads not a multiple of the 4 warps of a block."""
    _check("temporal odd sites", rung, temporal_case(ops, rung, 1, T0, sites, 3, seed=sites), f"sites={sites}")


@pytest.mark.parametrize("rung", ["centred", "peaked16", "shift-30", "v-offset"])
def test_temporal_attn_level0(ops, rung):
    """The level-0 call: 9216 sites x 5 heads = 46080 pairs per batch element, past the 16 pairs per SM where the grid strides."""
    _check("temporal level0", rung, temporal_case(ops, rung, 2, T0, HW0, HEADS0, seed=43), "sites=9216")


# ------------------------------------------------------------------------------------------------ softmax_rows
SM_SCALE = 512 ** -0.5      # the VAE AttnBlock's C^-0.5


def softmax_scores(rung, rows, cols, seed):
    """fp32 [rows, cols] raw scores whose logits scores * SM_SCALE follow the rung."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = torch.randn(rows, cols, generator=g, device="cuda") / SM_SCALE
    if rung == "centred":
        return n
    if rung == "peaked":
        return 16.0 * n
    if rung == "offset+1000":
        return 1000.0 + n
    if rung == "sink":
        n[:, 0] += 15.0 / SM_SCALE
        return n
    if rung == "single":
        x = torch.full_like(n, -math.inf)
        j = torch.randint(0, cols, (rows,), generator=g, device="cuda")
        x[torch.arange(rows, device="cuda"), j] = n[:, 0]
        return x
    if rung == "equal":
        return torch.full_like(n, 3.7)
    raise ValueError(rung)


SM_RUNGS = ["centred", "peaked", "offset+1000", "sink", "single", "equal"]


def _softmax_check(ops, rung, x, what):
    p = ops.softmax_rows(x, SM_SCALE)
    _check("softmax_rows", rung, ar.worst_ratio(p, ar.softmax_ref(x, SM_SCALE), ar.softmax_bound(x, SM_SCALE)), what)


@pytest.mark.parametrize("rung", SM_RUNGS)
@pytest.mark.parametrize("cols", [1, 255, 256, 257, 1000, 9216])
def test_softmax_rows(ops, cols, rung):
    _softmax_check(ops, rung, softmax_scores(rung, 64, cols, cols), f"cols={cols}")


@pytest.mark.parametrize("rung", SM_RUNGS)
def test_softmax_rows_padded_keys(ops, rung):
    """A 5x9 VAE latent: 45 tokens, the key axis padded to 48 with -inf."""
    x = torch.cat([softmax_scores(rung, 45, 45, 5), torch.full((45, 3), -math.inf, device="cuda")], 1)
    _softmax_check(ops, rung, x, "48 cols, 3 padded")


# ------------------------------------------------------------------------------------------------ VAE AttnBlock end to end
def _vae_block(logit_std, seed):
    """A seeded _VAttn(512) whose q / k weights are scaled so the logits of a GroupNorm-ed N(0,1) input have about `logit_std`."""
    from viewcrafter_b200.autoencoder import AutoencoderKL, _VAttn
    torch.manual_seed(seed)
    m = _VAttn(512)
    with torch.no_grad():
        m.norm.weight.copy_(1.0 + 0.2 * torch.randn(512))
        m.norm.bias.copy_(0.2 * torch.randn(512))
        hn = torch.randn(256, 512, dtype=torch.float64) * m.norm.weight.double() + m.norm.bias.double()
        wq, wk = m.q.weight.double().reshape(512, 512), m.k.weight.double().reshape(512, 512)
        s = (hn @ wq.t() + m.q.bias.double()) @ (hn @ wk.t() + m.k.bias.double()).t() * SM_SCALE
        f = math.sqrt(logit_std / float(s.std()))
        for lin in (m.q, m.k):
            lin.weight.mul_(f)
            lin.bias.mul_(f)
    return AutoencoderKL._pack_attn(SimpleNamespace(_f32=AutoencoderKL._f32), m.cuda())


def vae_attn_ref(P, x):
    """float64 AttnBlock on x [HW, 512] fp16 with P's fp16 weights, and two error bounds of the fused chain, which rounds GroupNorm's
    output (fp16; mean and rstd within the 2e-4 the norm-statistics tests hold), q, k and V^T (fp16, fp32 accumulation over 512), the
    probabilities (`softmax_bound`), P V + b_v (fp16, fp32 accumulation over the keys) and proj_out + residual (fp16).  A logit error
    ds_ij moves o_i by sum_j p_ij ds_ij (v_j - o_i).

    bound: first-order worst case, each rounding at its bound and carried through |W|.  It holds for every element but adds |W| |x|
    where the error adds W x, about 18x too much per 512-wide GEMM, so it only catches gross mistakes.
    sigma: every rounding is an independent zero-mean error of variance at most (its bound)^2 / 3 (uniform), carried through W^2; the
    RMS error of the block is at most the RMS of sigma.  Returns (y, bound, sigma, y - x)."""
    u, u2, g23 = ar.U, ar.U ** 2 / 3, 2.0 ** -23
    HW, C = x.shape
    xd = x.double()
    gamma, beta = (t.double() for t in P["gn"])
    xv = xd.view(HW, 32, C // 32)
    mean = xv.mean(dim=(0, 2), keepdim=True)
    rstd = 1.0 / torch.sqrt((xv - mean).square().mean(dim=(0, 2), keepdim=True) + 1e-6)
    xhat = ((xv - mean) * rstd).view(HW, C)
    h = xhat * gamma + beta
    gn_err = 2e-4 * gamma.abs() * (xhat.abs() + 1.0)
    dh, var_h = u * h.abs() + gn_err + 2.0 ** -24, u2 * h.square() + gn_err.square() / 3
    wq, wk = P["qk_w"].double()[:C], P["qk_w"].double()[C:]
    bq, bk = P["qk_b"].double()[:C], P["qk_b"].double()[C:]
    wv, wo = P["v_w"].double(), P["o_w"].double()
    gk = C * g23
    q, k, v = h @ wq.t() + bq, h @ wk.t() + bk, h @ wv.t()
    dq, dk, dv = (u * t.abs() + (dh + gk * h.abs()) @ w.abs().t() + 2.0 ** -24 for t, w in ((q, wq), (k, wk), (v, wv)))
    var_q, var_k, var_v = (u2 * t.square() + var_h @ w.square().t() for t, w in ((q, wq), (k, wk), (v, wv)))
    o, do, var_o = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
    mu = v.mean(0, keepdim=True)
    gkv = ((HW + 7) // 8 * 8) * g23
    step = max(1, CHUNK // (2 * HW))
    for r0 in range(0, HW, step):
        rs = slice(r0, r0 + step)
        raw = q[rs] @ k.t()
        p = torch.softmax(raw * SM_SCALE, -1)
        sb = ar.softmax_bound(raw, SM_SCALE)
        oc = p @ v
        o[rs] = oc + P["v_b"].double()
        w = p * SM_SCALE * (dq[rs] @ k.abs().t() + q[rs].abs() @ dk.t() + gk * (q[rs].abs() @ k.abs().t()))
        do[rs] = (u * o[rs].abs() + p @ dv + sb @ v.abs() + w @ (v - mu).abs() + (oc - mu).abs() * w.sum(-1, keepdim=True)
                  + gkv * (p @ v.abs()) + 2.0 ** -24)
        w = p.square() * SM_SCALE ** 2 * (var_q[rs] @ k.square().t() + q[rs].square() @ var_k.t())
        spread = (w @ v.square() - 2 * oc * (w @ v) + oc.square() * w.sum(-1, keepdim=True)).clamp_min(0)
        var_o[rs] = u2 * o[rs].square() + p.square() @ var_v + sb.square() @ v.square() / 3 + spread
    branch = o @ wo.t() + P["o_b"].double()
    y = xd + branch
    bound = (u * y.abs() + (do + gk * o.abs()) @ wo.abs().t() + 2.0 ** -24) * (1 + 2.0 ** -10)
    sigma = (u2 * y.square() + var_o @ wo.square().t()).sqrt()
    return y, bound, sigma, branch


@pytest.mark.parametrize("logit_std", [1.0, 8.0])
@pytest.mark.parametrize("H,W", [(72, 128), (5, 9)])
def test_vae_attnblock(ops, H, W, logit_std):
    """AutoencoderKL._attn on one image against an fp64 AttnBlock, within both bounds of `vae_attn_ref`."""
    from viewcrafter_b200.autoencoder import AutoencoderKL
    P = _vae_block(logit_std, 5)
    HW = H * W
    x = torch.randn(HW, 512, generator=torch.Generator(device="cuda").manual_seed(6), device="cuda").half()
    y = AutoencoderKL._attn(P, x, 1, H, W)
    ref, bound, sigma, branch = vae_attn_ref(P, x)
    assert bool(torch.isfinite(y).all())
    err = (y.double() - ref).abs()
    rms_branch = float(branch.square().mean().sqrt())
    rel_rms, rel_rms_bound = float(err.square().mean().sqrt()) / rms_branch, float(sigma.square().mean().sqrt()) / rms_branch
    max_ratio = float((err / bound).max())
    rung = f"{H}x{W} std{logit_std:g}"
    _note("vae attnblock max", rung, max_ratio)
    _note("vae attnblock rel-rms", rung, rel_rms / rel_rms_bound)
    print(f"\nVAE AttnBlock {rung}: max |y - ref| / bound {max_ratio:.3g}, relative RMS error {rel_rms:.3g} (bound {rel_rms_bound:.3g})")
    assert max_ratio <= 1.0
    assert rel_rms <= rel_rms_bound


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--bn64", type=int, choices=[0, 1], required=True, help="1: 64-key tiles for every shape, 0: 128-key tiles")
    sys.exit(_forced_main(ap.parse_args().bn64))
