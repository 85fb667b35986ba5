"""Every place the forward takes GroupNorm / LayerNorm statistics from, on offset and degenerate activations, against float64.

Centred Gaussian data cannot tell a one-pass ``E[x^2] - mean^2`` variance from a correct one, so each statistics path runs on a ladder
of rungs: centred, row / group means of 16, 64 and 256 standard deviations, per-channel offsets inside a group, large magnitudes, a
variance below eps (at both eps values the model uses) and constant rows / groups.  The reference is one float64 helper (`norm_ref`)
applied to the fp16 input as stored; no kernel is compared with another.

Bounds: normalised fp16 outputs |y - ref| <= 3e-3 + 4e-3 |ref|; returned statistics: rstd relative error <= 2e-4 and
|mean error| * rstd <= 2e-4; constant rows: rstd == eps^-0.5 to 1e-6.  LayerNorm paths hold them on every rung.  The GroupNorm paths
keep (sum, sumsq) records and hold the output bound on every group whose |mean| / std <= 64; the other groups (the mu256 and tiny rungs,
constant groups) get a loose regression bound (about a 5 % rstd error).  The worst errors per path and rung are printed at the end of the
module: run with ``-s`` to see the table.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.norm_rungs import REPORT, RUNGS, RUNGS_EPS5, _gen, _gn_check, _note, affine, check_out, check_stats, norm_ref, rung_data  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module", autouse=True)
def _report():
    REPORT.clear()          # shared with the other modules that use the ladder: print this module's rows only
    yield
    if not REPORT:
        return
    keys = ["out/bound", "loose out/bound", "rstd_rel", "mean*rstd"]
    print("\nworst error per path and rung (out/bound: max |y - ref| / (3e-3 + 4e-3 |ref|), <= 1 passes; loose: GroupNorm groups with "
          "|mean| > 64 std)")
    print(f"{'path':34s} {'rung':14s} " + " ".join(f"{k:>15s}" for k in keys))
    for (path, rung), d in sorted(REPORT.items()):
        print(f"{path:34s} {rung:14s} " + " ".join(f"{d[k]:15.3g}" if k in d else f"{'-':>15s}" for k in keys))


# ------------------------------------------------------------------------------------------------ 1. layernorm (layernorm_kernel<2/5/8>)
@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("C", [64, 512, 520, 1280, 1288, 2048])
def test_layernorm_rows(ops, C, rung):
    eps = RUNGS[rung][0]
    g, b = affine(C, 1)
    for rows in (1, 7, 1000):
        x = rung_data(rung, rows, C, seed=rows + C)
        ref, _, _ = norm_ref(x, g, b, eps)
        check_out("1 layernorm", rung, ops.layernorm(x, g, b, eps), ref)


# ------------------------------------------------------------------------------------------------ 2. layernorm_stats (pivoted one pass)
@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("C", [320, 512, 1024, 1032, 2560])
def test_layernorm_stats(ops, C, rung):
    eps = RUNGS[rung][0]
    for rows in (1, 7, 1003):
        x = rung_data(rung, rows, C, seed=3 * rows + C)
        st = ops.layernorm_stats(x, eps)
        _, mean, rstd = norm_ref(x, torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), eps)
        check_stats("2 layernorm_stats", rung, st[:, 0], st[:, 1], mean, rstd, eps)


# ------------------------------------------------------------------------------------------------ 3. LayerNorm statistics from the GEMM
def _producer(rung, M, N, seed, res):
    """(x, w, bias, r) of a linear whose output is on the rung.  With a residual the offset enters through it, as in a transformer block's
    residual stream, and the GEMM adds a small term (none for the tiny / constant rungs); without one, w is the identity and x the rung."""
    if not res:
        return rung_data(rung, M, N, seed), torch.eye(N, device="cuda", dtype=torch.float16), None, None
    K = 320
    x = rung_data("centred", M, K, seed + 1)
    quiet = rung.startswith(("tiny", "const"))
    w = (torch.randn(N, K, generator=_gen(seed + 2), device="cuda") * (0.0 if quiet else 0.3 * K ** -0.5)).half()
    bias = None if quiet else 0.1 * torch.randn(N, generator=_gen(seed + 3), device="cuda")
    return x, w, bias, rung_data(rung, M, N, seed + 4)


@pytest.mark.parametrize("rung", RUNGS_EPS5)
@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("N", [320, 640, 1280])
def test_linear_ln_out_statistics(ops, N, res, rung):
    """linear(..., ln_out=True): the (mean, rstd) of the stored output, from the epilogue's per-32-column records."""
    M = 1000
    x, w, bias, r = _producer(rung, M, N, seed=N, res=res)
    y, st = ops.linear(x, w, bias=bias, res=r, ln_out=True)
    assert torch.equal(y, ops.linear(x, w, bias=bias, res=r)), "ln_out changed the output"
    _, mean, rstd = norm_ref(y, torch.ones(N, device="cuda"), torch.zeros(N, device="cuda"), 1e-5)
    check_stats("3 linear ln_out", rung, st[:, 0], st[:, 1], mean, rstd, 1e-5)


@pytest.mark.parametrize("rung", [r for r in RUNGS_EPS5 if not r.startswith("const")])
@pytest.mark.parametrize("N", [320, 640, 1280])
def test_ln_out_folded_into_next_linear(ops, N, rung):
    """x, st = linear(..., res=h, ln_out=True) -> linear(x, fold_layernorm(...), ln=(st, cs)) (and the GEGLU form) against float64
    LayerNorm -> Linear (-> GEGLU) of x as stored: a transformer block's residual GEMM feeding the next folded LayerNorm.  Not on
    constant rows: the folded form rstd * (W'x - mean * colsum) multiplies the fp32 rounding of W'x by eps^-1/2 = 316 there (the
    statistics of constant rows are checked above)."""
    M = 700
    a, w1, b1, h = _producer(rung, M, N, seed=7 * N, res=True)
    x, st = ops.linear(a, w1, bias=b1, res=h, ln_out=True)
    g = _gen(11)
    gamma = 2.0 ** torch.randint(-1, 2, (N,), generator=g, device="cuda").float()    # powers of two: the fold's fp16 W * gamma is exact
    beta = 0.3 * torch.randn(N, generator=g, device="cuda")
    xn, _, _ = norm_ref(x, gamma, beta, 1e-5)
    # Linear
    w = (torch.randn(N, N, generator=g, device="cuda") * N ** -0.5).half().float()
    bias = 0.2 * torch.randn(N, generator=g, device="cuda")
    w16, cs, b2 = ops.fold_layernorm(w, gamma, beta, bias)
    out = ops.linear(x, w16, bias=b2, ln=(st, cs))
    ref = xn @ w.double().t() + bias.double()
    err = (out.double() - ref).abs()
    _note("3 ln_out -> folded linear", rung, **{"out/bound": float((err / (6e-3 + 4e-3 * ref.abs())).max())})
    assert bool((err <= 6e-3 + 4e-3 * ref.abs()).all()), f"folded linear {rung}: max err {float(err.max()):.4g}"
    # GEGLU
    wg = (torch.randn(8 * N, N, generator=g, device="cuda") * N ** -0.5).half().float()
    bg = 0.1 * torch.randn(8 * N, generator=g, device="cuda")
    wp, bp, csg = ops.pack_geglu_ln(wg, bg, gamma, beta)
    out = ops.linear(x, wp, bias=bp, geglu=True, ln=(st, csg))
    hh = xn @ wg.double().t() + bg.double()
    val, gate = hh.chunk(2, dim=-1)
    ref = val * F.gelu(gate)
    err = (out.double() - ref).abs()
    _note("3 ln_out -> folded geglu", rung, **{"out/bound": float((err / (8e-3 + 4e-3 * ref.abs())).max())})
    assert bool((err <= 8e-3 + 4e-3 * ref.abs()).all()), f"folded geglu {rung}: max err {float(err.max()):.4g}"


# ------------------------------------------------------------------------------------------------ 4. groupnorm, statistics pass
GN_SHAPES = [  # samples, rows per sample, C, silu
    (1, 1, 32, False), (5, 1, 2560, True), (5, 33, 64, True), (1, 33, 1280, False), (5, 33, 320, False),
    (1, 9216, 320, True), (5, 9216, 64, False), (1, 9216, 2560, False), (5, 9216, 1280, True),
    (1, 576 * 1024, 128, True),        # a VAE decoder GroupNorm: one 576x1024 frame
]


@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("samples,rows,C,silu", GN_SHAPES)
def test_groupnorm_statistics_pass(ops, samples, rows, C, silu, rung):
    eps = RUNGS[rung][0]
    x = rung_data(rung, samples * rows, C, seed=rows + C, samples=samples)
    gamma, beta = affine(C, 2)
    _gn_check("4 groupnorm", rung, ops.groupnorm(x, samples, gamma, beta, eps, silu), x, samples, gamma, beta, eps, silu)


@pytest.mark.parametrize("rung", list(RUNGS))
def test_groupnorm_concat_statistics_pass(ops, rung):
    """[x1 | x2] with x1 at +20 and x2 at -20 (on top of the rung): C1 = 640, C2 = 320 gives 30-channel groups, one of them straddles
    the concat boundary and its variance holds the 40-unit step."""
    eps = RUNGS[rung][0]
    samples, rows = 3, 576
    x1 = (rung_data(rung, samples * rows, 640, seed=21, samples=samples).float() + 20.0).half()
    x2 = (rung_data(rung, samples * rows, 320, seed=22, samples=samples).float() - 20.0).half()
    gamma, beta = affine(960, 3)
    out = ops.groupnorm(x1, samples, gamma, beta, eps, True, x2=x2)
    _gn_check("4 groupnorm concat", rung, out, torch.cat([x1, x2], 1), samples, gamma, beta, eps, True)


# ------------------------------------------------------------------------------------------------ 5. groupnorm from the GEMM's gn_part records
def _force_gn_parts(ops, monkeypatch):
    monkeypatch.setattr(ops, "GN_FROM_PRODUCER", 2)
    monkeypatch.setattr(ops, "GN_PARTS_MIN_MB", 0.0)


def _quiet(rung):
    return 0.0 if rung.startswith(("tiny", "const")) else 1.0


@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("producer", ["conv3x3", "conv_temporal", "linear"])
def test_groupnorm_from_producer_records(ops, monkeypatch, producer, rung):
    """GroupNorm of a GEMM output that carries its gn_part records, per frame (4-D) and per batch element (5-D); the rung enters through
    the residual."""
    _force_gn_parts(ops, monkeypatch)
    eps = RUNGS[rung][0]
    B, T, H, W, Ci, C = 2, 4, 18, 32, 64, 320
    M = B * T * H * W
    g = _gen(31)
    x = rung_data("centred", M, Ci, seed=32)
    r = rung_data(rung, M, C, seed=33, samples=B * T)
    s = 0.3 * _quiet(rung)
    if producer == "conv3x3":
        w = ops.pack_conv3x3(torch.randn(C, Ci, 3, 3, generator=g, device="cuda") * s / math.sqrt(9 * Ci))
        y = ops.conv3x3(x, B * T, H, W, w, res=r, gn_out=True)
    elif producer == "conv_temporal":
        x = rung_data("centred", M, C, seed=34)
        w = ops.pack_conv_temporal(torch.randn(C, C, 3, 1, 1, generator=g, device="cuda") * s / math.sqrt(3 * C))
        y = ops.conv_temporal(x, B, T, H * W, w, res=r, gn_out=True)
    else:
        y = ops.linear(x, (torch.randn(C, Ci, generator=g, device="cuda") * s / math.sqrt(Ci)).half(), res=r, gn_out=True)
    assert ops.gn_part_of(y) is not None
    gamma, beta = affine(C, 4)
    for samples, silu in ((B * T, True), (B, False)):
        n0 = ops.gn_from_parts_calls
        out = ops.groupnorm(y, samples, gamma, beta, eps, silu)
        assert ops.gn_from_parts_calls - n0 == 1, "expected the statistics from the producer's records"
        _gn_check(f"5 gn_part {producer} {'4-D' if samples == B * T else '5-D'}", rung, out, y, samples, gamma, beta, eps, silu)


@pytest.mark.parametrize("rung", list(RUNGS))
def test_groupnorm_concat_from_producer_records(ops, monkeypatch, rung):
    """The skip-concat GroupNorm from both producers' records: a linear's output at +20, a conv's at -20, 30-channel groups."""
    _force_gn_parts(ops, monkeypatch)
    eps = RUNGS[rung][0]
    frames, H, W = 3, 18, 32
    M = frames * H * W
    g = _gen(41)
    s = 0.3 * _quiet(rung)
    ra = (rung_data(rung, M, 640, seed=42, samples=frames).float() + 20.0).half()
    rb = (rung_data(rung, M, 320, seed=43, samples=frames).float() - 20.0).half()
    a = ops.linear(rung_data("centred", M, 64, seed=44), (torch.randn(640, 64, generator=g, device="cuda") * s / 8).half(), res=ra,
                   gn_out=True)
    wb = ops.pack_conv3x3(torch.randn(320, 64, 3, 3, generator=g, device="cuda") * s / 24)
    b = ops.conv3x3(rung_data("centred", M, 64, seed=45), frames, H, W, wb, res=rb, gn_out=True)
    gamma, beta = affine(960, 5)
    n0 = ops.gn_from_parts_calls
    out = ops.groupnorm(a, frames, gamma, beta, eps, True, x2=b)
    assert ops.gn_from_parts_calls - n0 == 1
    _gn_check("5 gn_part concat", rung, out, torch.cat([a, b], 1), frames, gamma, beta, eps, True)


# ------------------------------------------------------------------------------------------------ 6. reproducible mode: canonical leaves
@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("samples,rows,C1,C2", [(2, 9216, 320, 0), (5, 33, 64, 0), (3, 576, 640, 320)])
def test_groupnorm_canonical(ops, samples, rows, C1, C2, rung):
    eps = RUNGS[rung][0]
    x1 = rung_data(rung, samples * rows, C1, seed=51, samples=samples)
    x2 = None
    if C2:
        x1 = (x1.float() + 20.0).half()
        x2 = (rung_data(rung, samples * rows, C2, seed=52, samples=samples).float() - 20.0).half()
    gamma, beta = affine(C1 + C2, 6)
    prev = ops.set_reproducible(True)
    try:
        out = ops.groupnorm(x1, samples, gamma, beta, eps, True, x2=x2)
    finally:
        ops.set_reproducible(prev)
    x = x1 if x2 is None else torch.cat([x1, x2], 1)
    _gn_check("6 groupnorm_canonical", rung, out, x, samples, gamma, beta, eps, True)


# ------------------------------------------------------------------------------------------------ 7. split form of the multi-GPU GroupNorm
@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("samples,rows,C", [(2, 9216, 320), (1, 2 * 4608, 1280), (5, 66, 64)])
def test_groupnorm_split_statistics(ops, samples, rows, C, rung):
    """What a 2-rank all-reduce runs (parallel.py groupnorm5d): groupnorm_stats of each rank's half of every sample's rows, added, then
    groupnorm_apply of each half with the full row count.  The statistics the added (sum, sumsq) give are printed, and held to the
    regression bound."""
    eps = RUNGS[rung][0]
    x = rung_data(rung, samples * rows, C, seed=61, samples=samples)
    xs = x.view(samples, rows, C)
    halves = [xs[:, :rows // 2].reshape(-1, C).contiguous(), xs[:, rows // 2:].reshape(-1, C).contiguous()]
    st = ops.groupnorm_stats(halves[0], samples) + ops.groupnorm_stats(halves[1], samples)
    gamma, beta = affine(C, 7)
    outs = [ops.groupnorm_apply(h, samples, st, rows, gamma, beta, eps, False) for h in halves]
    out = torch.cat([o.view(samples, rows // 2, C) for o in outs], 1).view(-1, C)
    _gn_check("7 groupnorm split", rung, out, x, samples, gamma, beta, eps, False)
    # the statistics the apply pass forms from the records (fp64, as gn_apply_dev does)
    n = rows * (C // 32)
    s, q = st[..., 0].double(), st[..., 1].double()
    mean = s / n
    rstd = 1.0 / torch.sqrt((q / n - mean * mean).clamp_min(0.0) + eps)
    _, mean_ref, rstd_ref = norm_ref(x, torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), eps, samples=samples)
    rel = float(((rstd - rstd_ref) / rstd_ref).abs().max())
    dm = float(((mean - mean_ref).abs() * rstd_ref).max())
    _note("7 groupnorm split", rung, rstd_rel=rel, **{"mean*rstd": dm})
    if not rung.startswith("const"):         # a constant group's rstd is eps^-0.5 times whatever the rounding leaves of its variance
        assert rel <= 0.05, f"split statistics {rung}: rstd relative error {rel:.3g} (regression bound 5 %)"
