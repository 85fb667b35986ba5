"""The VAE at the frame sizes it runs at: 576x1024 (ViewCrafter_25) and 320x512 (ViewCrafter_25_512).

1. Its tap-GEMMs at the VAE's geometries against float64, with the bound of test_gemm_sweep_gpu.py (fp32 accumulation over K_total plus
   one rounding to the output type; the upsample-conv adds 2^-11 |A| @ |W|^T for its pre-summed parity taps).  These are the widths the
   small-geometry sweep does not reach: 128-pixel boxes with 1, 2, 4 and 8 boxes per image row at many tiles per CTA, the four parity
   stores of upconv3x3 at W = 64..512, conv_in's K = 8 after k_pad, the ragged N = 3 fp32 conv_out, the encoder's stride-2 downsample
   and the ResnetBlock's nin_shortcut residual as AutoencoderKL._res wires it.  Conv cases go through the sweep's Conv.check, which passes
   acc1: these cases feed the sweep's accumulation ratio, and test_report_accumulation_ratio below holds it to C_ACC.  GroupNorm (eps 1e-6,
   SiLU) at the VAE's shapes goes through the norm ladder's _gn_check.  The worst |out - ref| / bound per case is printed when the module
   ends (run with -s).  Short reductions (conv_in's K = 72, the 1x1 nin_shortcut) sit close to 1: there the output's own rounding, half an
   ulp, is nearly all of the bound.  Negative controls show the bound rejects the geometry bugs these cases are for.

2. AutoencoderKL.decode / encode_moments end to end against the oracle run on the GPU with the same weights, by the self-calibrating rule
   of test_zz_baseline_size_gpu.py:  E_ref = |oracle under torch.autocast(fp16) - oracle in fp32|,  accept when
   max|ours - fp32| <= 2 max E_ref  and  mean|ours - fp32| <= 2 mean E_ref.  The synthetic weights of oracle/synth.py are used unscaled
   (rounded to fp16 values, on both sides, so the kernel cases' float64 references use the packed weights exactly): the fp32 oracle's
   activations stay in the low hundreds, far from the fp16 range, and the test asserts the autocast output is finite.  The numbers are
   printed and written to $VC_PARITY_OUT/parity_vae_full_size.json when that variable names a directory.
"""
import json
import os
import time

import pytest
import torch
import torch.nn.functional as F

from tests.norm_rungs import REPORT as GN_REPORT
from tests.norm_rungs import _gn_check, affine, rung_data
from tests.test_gemm_sweep_gpu import (C_ACC, Conv, _outside, _randn, _rows, acc_err, bound_of, carve_a, carve_w, check, f16, f32,
                                       worst)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]

_T0 = time.time()
RATIO = {}                                               # case -> worst |out - ref| / bound
_RESULTS = {}                                            # end-to-end parity numbers


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def vae(ops):
    """(full-width AutoencoderKL on cuda, its state dict on cuda): synthetic weights rounded to fp16 values."""
    from oracle import synth
    from viewcrafter_b200.autoencoder import AutoencoderKL
    from viewcrafter_b200.configs import VAE_DDCONFIG
    m = AutoencoderKL(VAE_DDCONFIG, None, 4)
    sd = {k: v.half().float() for k, v in synth.synth_state_dict(synth.module_shapes(m), seed=51).items()}
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), {k: v.cuda() for k, v in sd.items()}


@pytest.fixture(scope="module", autouse=True)
def _report():
    GN_REPORT.clear()       # shared with the other modules that use the norm ladder: print this module's rows only
    yield
    if RATIO:
        print(f"\nVAE full size: worst |out - ref| / bound per case ({time.time() - _T0:.0f} s)")
        print(f"{'case':58s} {'worst |out-ref|/bound':>22s}")
        for k, v in RATIO.items():
            print(f"{k:58s} {v:22.3g}")
    if GN_REPORT:
        print("\nVAE GroupNorm (eps 1e-6, SiLU): out/bound = max |y - ref| / (3e-3 + 4e-3 |ref|); loose: groups with |mean| > 64 std")
        for (path, rung), d in sorted(GN_REPORT.items()):
            print(f"{path:34s} {rung:14s} " + " ".join(f"{k} {v:.3g}" for k, v in d.items()))
    if _RESULTS:
        print("\nVAE end to end vs the fp32 oracle (E_ref = |autocast - fp32|)")
        for k, r in _RESULTS.items():
            print(f"{k:34s} " + " ".join(f"{n} {v:.4g}" for n, v in r.items()))


def _note(case, out, ref, err):
    d = (out.double() - ref).abs()
    r = float((d / bound_of(ref, err, out.dtype)).nan_to_num(float("inf")).max())
    RATIO[case] = max(RATIO.get(case, 0.0), r)


def _check(out, ref, err, case):
    _note(case, out, ref, err)
    check(out, ref, err, case)


def _nchw(rows, frames, H, W):                           # [(n h w), c] -> float64 [n, c, h, w]
    return rows.view(frames, H, W, -1).permute(0, 3, 1, 2).double()


def _w64(conv):
    return conv.weight.detach().double()


def _b64(conv):
    return conv.bias.detach().double()


# ------------------------------------------------------------------------------------------------------------- conv3x3
class ConvIn(Conv):
    """conv_in: Ci = 3 or 4 input channels in 8-column rows whose other columns are zero (ncthw_to_rows into zeroed rows), weights
    packed by pack_conv3x3(k_pad=8): the GEMM runs K = 8."""

    def __init__(self, ops, frames, H, W, Ci, Co, seed):
        self.frames, self.H, self.W, self.Co, self.C2, self.bzd = frames, H, W, Co, 0, 0
        xi = _randn((frames, Ci, H, W), seed).half()
        wc = _randn((Co, Ci, 3, 3), seed + 1, (9 * Ci) ** -0.5).half()
        rows = torch.zeros(frames * H * W, 8, dtype=torch.float16)
        rows[:, :Ci] = _rows(xi)
        self.x, self.x2 = carve_a(rows.cuda()), None
        self.w9 = carve_w(ops.pack_conv3x3(wc, k_pad=8).cuda(), pitched=False)
        self.b, self.M, self.r = f32((Co,), seed + 2), frames * H * W, None
        x64, w64 = xi.double().cuda(), wc.double().cuda()
        self.mm = _rows(F.conv2d(x64, w64, padding=1))
        self.absacc = _rows(F.conv2d(x64.abs(), w64.abs(), padding=1))
        self.k_total = 9 * 8


def _run_conv(ops, case, name, out_kind="f16", res_kind="contig"):
    out = case.check(ops, name, out_kind=out_kind, res_kind=res_kind)
    ref, err, _ = case.ref(with_res=res_kind is not None)
    _note(name, out, ref, err)


@pytest.mark.parametrize("frames,H,W,Ci,Co", [(2, 72, 128, 4, 512), (1, 576, 1024, 3, 128)])
def test_conv_in(ops, frames, H, W, Ci, Co):
    """decoder conv_in (4 latent channels, 72x128) and encoder conv_in (3 colour channels, 576x1024)"""
    _run_conv(ops, ConvIn(ops, frames, H, W, Ci, Co, seed=100 + Ci), f"conv_in {frames}x{H}x{W} {Ci}(k_pad 8)->{Co}", res_kind=None)


# 1, 2, 4 and 8 128-pixel boxes per image row; 40x64 is the 320x512 workload's latent (64x2 boxes)
CONV_RES = [(2, 72, 128, 512, 512), (2, 144, 256, 512, 512), (2, 288, 512, 512, 256), (2, 288, 512, 256, 256),
            (1, 576, 1024, 256, 128), (1, 576, 1024, 128, 128), (2, 40, 64, 512, 512)]


@pytest.mark.parametrize("frames,H,W,Ci,Co", CONV_RES)
def test_conv3x3_residual(ops, frames, H, W, Ci, Co):
    case = Conv(frames, H, W, Ci, Co, seed=200 + W + Ci + Co)
    _run_conv(ops, case, f"conv3x3+res {frames}x{H}x{W} {Ci}->{Co}")


@pytest.mark.parametrize("frames,H,W,Ci,Co,what", [(1, 576, 1024, 128, 3, "decoder conv_out"),
                                                   (2, 72, 128, 512, 8, "encoder conv_out.quant_conv")])
def test_conv3x3_f32_out(ops, frames, H, W, Ci, Co, what):
    """fp32 output with a ragged N (3 or 8 columns), contiguous and through a pitched view (pitch % 8 == 3)"""
    case = Conv(frames, H, W, Ci, Co, seed=300 + Co, res=False)
    for ok in ("f32", "f32_p3"):
        _run_conv(ops, case, f"{what} {frames}x{H}x{W} {Ci}->{Co} {ok}", out_kind=ok, res_kind=None)


# ------------------------------------------------------------------------------------------------------------- upsample-conv
def upconv_ref(x64, w64, b):
    """float64 conv3x3(upsample2x(x)) + bias, and the bound of the parity GEMMs (taps of 4 Ci, pre-summed fp16 weights)"""
    xu = F.interpolate(x64, scale_factor=2, mode="nearest")
    ref = _rows(F.conv2d(xu, w64, padding=1)) + b.double()
    absacc = _rows(F.conv2d(xu.abs(), w64.abs(), padding=1))
    return ref, acc_err(4 * x64.shape[1], absacc, b.double().abs()) + 2.0 ** -11 * absacc


@pytest.mark.parametrize("lvl,frames,H,W", [(3, 2, 72, 128), (2, 2, 144, 256), (1, 1, 288, 512), (3, 2, 40, 64)])
def test_upconv3x3(ops, vae, lvl, frames, H, W):
    """The decoder's Upsample convs with their packed weights, at W = 128 / 256 / 512 (1, 2, 4 boxes per row) and at the 320x512
    workload's 40x64 -> 80x128 (64x2 boxes): every parity's stores through ldo = 2N, ldo_y = 4WN, ldo_z = 4WHN."""
    m, _ = vae
    P = m._packed or m._pack()
    S, conv = P["up"][lvl], m.decoder.up[lvl].upsample.conv
    C = conv.in_channels
    x = _randn((frames, C, H, W), 400 + lvl + W).half()
    y = ops.upconv3x3(carve_a(_rows(x).cuda()), frames, H, W, [carve_w(p, pitched=False) for p in S["up_w"]], bias=S["up_b"])
    ref, err = upconv_ref(x.double().cuda(), _w64(conv), S["up_b"])
    _check(y, ref, err, f"upconv3x3 {frames}x{H}x{W} -> {2 * H}x{2 * W} {C}")


# ------------------------------------------------------------------------------------------------------------- downsample
@pytest.mark.parametrize("lvl,frames,H,W", [(0, 1, 576, 1024), (1, 2, 288, 512), (2, 2, 144, 256)])
def test_downsample(ops, vae, lvl, frames, H, W):
    """The encoder's Downsample as it runs: im2col_s2(pad_lo=0, pad_hi=1) + linear with the packed weights, against
    conv2d(pad(x, (0, 1, 0, 1)), stride=2)."""
    m, _ = vae
    P = m._packed_enc or m._pack_encoder()
    S, conv = P["down"][lvl], m.encoder.down[lvl].downsample.conv
    C = conv.in_channels
    x = _randn((frames, C, H, W), 500 + lvl).half()
    cols, Ho, Wo = ops.im2col_s2(_rows(x).contiguous().cuda(), frames, H, W, pad_lo=0, pad_hi=1)
    assert (Ho, Wo) == (H // 2, W // 2)
    y = ops.linear(cols, carve_w(S["down_w"]), bias=S["down_b"])
    xp, w64 = F.pad(x.double().cuda(), (0, 1, 0, 1)), _w64(conv)
    ref = _rows(F.conv2d(xp, w64, stride=2)) + S["down_b"].double()
    absacc = _rows(F.conv2d(xp.abs(), w64.abs(), stride=2))
    _check(y, ref, acc_err(9 * C, absacc, S["down_b"].double().abs()), f"downsample {frames}x{H}x{W} -> {Ho}x{Wo} {C}")


# ------------------------------------------------------------------------------------------------------------- ResnetBlock
def _conv_ref(a_rows, frames, H, W, conv):
    a64, w64 = _nchw(a_rows, frames, H, W), _w64(conv)
    ref = _rows(F.conv2d(a64, w64, padding=1)) + _b64(conv)
    absacc = _rows(F.conv2d(a64.abs(), w64.abs(), padding=1))
    return ref, absacc


@pytest.mark.parametrize("lvl,H,W", [(1, 288, 512), (0, 576, 1024)])
def test_resnet_block_with_nin_shortcut(ops, vae, monkeypatch, lvl, H, W):
    """The first ResnetBlock of decoder levels 1 (512 -> 256 at 288x512, 147,456 rows) and 0 (256 -> 128 at 576x1024, 589,824 rows)
    through AutoencoderKL._res, one frame.  Every kernel call is recorded and checked against float64 from its recorded input:
    GroupNorm + SiLU, conv1, the 1x1 nin_shortcut linear, and conv2 plus the block's shortcut, which by the block's definition is the
    nin_shortcut output -- whatever residual conv2 was given."""
    from viewcrafter_b200.autoencoder import AutoencoderKL
    m, _ = vae
    P = m._packed or m._pack()
    Pb, blk = P["up"][lvl]["blocks"][0], m.decoder.up[lvl].block[0]
    Ci, Co = blk.conv1.in_channels, blk.conv1.out_channels
    assert "skip_w" in Pb and Ci != Co
    calls = []
    for name in ("groupnorm", "conv3x3", "linear"):
        def rec(*a, _fn=getattr(ops, name), _name=name, **k):
            y = _fn(*a, **k)
            calls.append((_name, y))
            return y
        monkeypatch.setattr(ops, name, rec)
    x = f16((H * W, Ci), 600 + lvl)
    y = AutoencoderKL._res(Pb, x, 1, H, W)
    monkeypatch.undo()
    assert [c[0] for c in calls] == ["groupnorm", "conv3x3", "groupnorm", "linear", "conv3x3"]
    a, h, b, xs = (c[1] for c in calls[:4])
    tag = f"{H}x{W} {Ci}->{Co}"
    for nm, out, inp in (("gn1", a, x), ("gn2", b, h)):
        gn = getattr(blk, "norm1" if nm == "gn1" else "norm2")
        _gn_check(f"block {nm} {tag}", "block", out, inp, 1, gn.weight.detach().float(), gn.bias.detach().float(), 1e-6, True)
    ref, absacc = _conv_ref(a, 1, H, W, blk.conv1)
    _check(h, ref, acc_err(9 * Ci, absacc, _b64(blk.conv1).abs()), f"block conv1 {tag}")
    ws, bs = _w64(blk.nin_shortcut).flatten(1), _b64(blk.nin_shortcut)
    x64 = x.double()
    _check(xs, x64 @ ws.t() + bs, acc_err(Ci, x64.abs() @ ws.abs().t(), bs.abs()), f"block nin_shortcut linear {H * W} x {Ci}->{Co}")
    ref, absacc = _conv_ref(b, 1, H, W, blk.conv2)
    extra = _b64(blk.conv2).abs() + xs.double().abs()
    _check(y, ref + xs.double(), acc_err(9 * Co, absacc, extra), f"block conv2 + nin_shortcut residual {tag}")


# ------------------------------------------------------------------------------------------------------------- GroupNorm
GN_SHAPES = [(2, 576 * 1024, 256), (2, 288 * 512, 512), (2, 144 * 256, 512), (1, 320 * 512, 128)]
GN_RUNGS = ["centred", "mu16", "mu64", "chan50", "tiny-eps1e-6", "const-eps1e-6"]


@pytest.mark.parametrize("rung", GN_RUNGS)
@pytest.mark.parametrize("samples,rows,C", GN_SHAPES)
def test_groupnorm_silu(ops, samples, rows, C, rung):
    x = rung_data(rung, samples * rows, C, seed=rows + C, samples=samples)
    gamma, beta = affine(C, 3)
    out = ops.groupnorm(x, samples, gamma, beta, 1e-6, True)
    _gn_check(f"gn {samples}x{rows}x{C}", rung, out, x, samples, gamma, beta, 1e-6, True)


# ------------------------------------------------------------------------------------------------------------- negative controls
def test_tolerance_rejects_vae_geometry_bugs(ops):
    """Reference side only, at the widths and channel counts of the cases above: each perturbed reference a geometry bug would produce
    falls outside the bound somewhere."""
    conv = Conv(1, 4, 1024, 128, 128, seed=700)
    ref, err, _ = conv.ref()
    bound = bound_of(ref, err, torch.float16)
    img = ref.view(1, 4, 1024, 128)
    box = img.clone()
    box[0, 2, 384:512] = img[0, 2, 512:640]                                  # one row's box 3 holds box 4's pixels
    assert _outside(box.view_as(ref), ref, bound), "128-pixel box column taken from the neighbouring box"
    shifted = torch.cat([img[:, :1], img[:, :-1]], 1)
    assert _outside(shifted.view_as(ref), ref, bound), "output shifted by one image row"
    x64 = _randn((1, 512, 3, 128), 701).half().double().cuda()
    w64 = _randn((512, 512, 3, 3), 702, (9 * 512) ** -0.5).half().double().cuda()
    uref, uerr = upconv_ref(x64, w64, f32((512,), 703))
    up = uref.view(1, 6, 256, 512)
    swapped = up.clone()
    swapped[:, 0::2, 1::2], swapped[:, 1::2, 0::2] = up[:, 1::2, 0::2], up[:, 0::2, 1::2]
    assert _outside(swapped.view_as(uref), uref, bound_of(uref, uerr, torch.float16)), "parities (0, 1) and (1, 0) swapped"
    blk = Conv(1, 4, 1024, 128, 128, seed=704, res=False)                    # conv2 of a 256 -> 128 block ...
    a = f16((4 * 1024, 256), 705)                                            # ... and its nin_shortcut, rounded to fp16
    ws, bs = f16((128, 256), 706, 256 ** -0.5).double(), f32((128,), 707).double()
    xs = (a.double() @ ws.t() + bs).half().double()
    bref, berr, _ = blk.ref()
    bref, berr = bref + xs, berr + acc_err(blk.k_total, 0, xs.abs())
    assert _outside(bref - xs, bref, bound_of(bref, berr, torch.float16)), "skip residual omitted"


# ------------------------------------------------------------------------------------------------------------- end to end
def _dump():
    out = os.environ.get("VC_PARITY_OUT")
    if not out:
        return
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "parity_vae_full_size.json"), "w") as f:
            json.dump(_RESULTS, f, indent=1)
    except OSError:
        pass


def _parity(key, fn, sd, inp, ours):
    """Run the oracle function twice on the GPU (fp32, autocast fp16) and apply the self-calibrating rule to ours."""
    from oracle import lvdm_oracle as O
    with torch.no_grad(), O.exact_fp32():
        ref32 = fn(sd, inp)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        ref16 = fn(sd, inp).float()
    ours = ours.float()
    assert ours.shape == ref32.shape, (key, ours.shape, ref32.shape)
    for nm, t in (("ours", ours), ("fp32 oracle", ref32), ("autocast oracle", ref16)):
        assert bool(torch.isfinite(t).all()), f"{key}: non-finite values in the {nm} output"
    e_ref, err = (ref16 - ref32).abs(), (ours - ref32).abs()
    r = dict(max_abs_err=float(err.max()), mean_abs_err=float(err.mean()), e_ref_max=float(e_ref.max()),
             e_ref_mean=float(e_ref.mean()), out_std=float(ref32.std()), out_absmax=float(ref32.abs().max()))
    _RESULTS[key] = r
    print(key, r)
    _dump()
    assert r["e_ref_max"] > 0 and r["e_ref_mean"] > 0, (key, r)
    assert r["max_abs_err"] <= 2.0 * r["e_ref_max"], (key, r)
    assert r["mean_abs_err"] <= 2.0 * r["e_ref_mean"], (key, r)


SIZES = {"ViewCrafter_25": (576, 1024), "ViewCrafter_25_512": (320, 512)}


@pytest.mark.parametrize("name", list(SIZES))
def test_decode_vs_oracle(vae, name):
    """AutoencoderKL.decode of 2 latents at 72x128 / 40x64"""
    from oracle import lvdm_oracle as O
    m, sd = vae
    H, W = SIZES[name]
    z = torch.randn(2, 4, H // 8, W // 8, generator=torch.Generator().manual_seed(800 + H)).cuda()
    _parity(f"decode {name}", O.vae_decode, sd, z, m.decode(z))


@pytest.mark.parametrize("name", list(SIZES))
def test_encode_moments_vs_oracle(vae, name):
    """AutoencoderKL.encode_moments of 2 frames at 576x1024 / 320x512"""
    from oracle import lvdm_oracle as O
    m, sd = vae
    H, W = SIZES[name]
    x = (torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(900 + H)) * 2 - 1).cuda()
    _parity(f"encode_moments {name}", O.vae_encode_moments, sd, x, m.encode_moments(x))


def test_report_accumulation_ratio(ops):
    """The conv cases above passed acc1 to the sweep's check: they hold its C_ACC, too.  The ratio is the sweep module's, so in a session
    that also ran test_gemm_sweep_gpu.py it covers those cases as well."""
    print(f"VAE full size: worst accumulation ratio {worst['ratio']:.4g} (C_ACC = {C_ACC})")
    assert worst["ratio"] <= C_ACC
