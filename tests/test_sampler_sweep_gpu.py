"""The fused sampler updates (ops.ddim_update, ops.dpm_update) on the step scalars the samplers really use, against the fp64
restatement of tests/test_dpm_solver_cpu.py, and the eta = 1 DDIM samplers end to end where 1 - a' - sigma^2 rounds below zero.

  * every step of every S in 1..100 (tests/test_sampler_sweep_cpu.step_counts), uniform_trailing and uniform spacing, base_scale 0.3 /
    0.7 (dynamic rescale on), eta 0 / 1, with two-way guidance at 7.5: the scalars come from DDIMSampler.step_scalars and
    DPMSolverSampler.step_scalars (c_hist from the solver's table), and a first-order DPM step must equal the DDIM update bit for bit;
  * the whole guidance grid -- two- / three-way (the ddim_multiplecond samplers' scalars) x guidance_rescale 0 / 0.7 -- at CFG_STEPS;
  * DDIMSampler and the three-way DDIMSampler at S = 4 and 25, eta = 1, finite; at S = 4 (where the reference's own fp32 radicand is
    >= 0) against the oracle's DDIM loop within the bounds of test_ddim_sample_three_steps_vs_oracle.
Every output must be finite and within 16 fp32 ulps of the magnitude of the terms it sums (test_dpm_solver_gpu.py's bound), times the
dynamic-rescale ratio prev_scale_t / scale_t where that is above 1 (pred_x0 is multiplied by it); x_prev also within the error of
sqrt(1 - a' - sigma^2) times |e_t| (_dir_error), which matters only at the first eta = 1 step, where that square root is taken of a
rounding error.
"""
import math

import pytest
import torch

from tests.test_dpm_solver_cpu import dpm_update_f64
from tests.test_sampler_sweep_cpu import BASE_SCALES, CFG_STEPS, E2E_STEPS, SPACINGS, ScheduleModel, sampler_steps, step_counts

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
EPS32 = 2.0 ** -23
N = 4 * 5 * 8 * 16 + 3                 # several 256-thread blocks and an odd tail
CFG, CFG_IMG = 7.5, 2.0


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _inputs():
    g = torch.Generator().manual_seed(5)
    cpu = [torch.randn(N, generator=g) * s for s in (1.0, 1.0, 1.2, 1.1, 1.0, 0.9)]     # x, v_cond, v_uncond, v_uncond_img, noise, x0_hist
    return cpu, [t.cuda() for t in cpu]


def _samplers(three_way, base_scale):
    from viewcrafter_b200 import ddim, ddim_multiplecond, dpm_solver
    m = ScheduleModel(base_scale)
    if three_way:
        return ddim_multiplecond.DDIMSampler(m), dpm_solver.DPMSolverSamplerMultiCond(m)
    return ddim.DDIMSampler(m), dpm_solver.DPMSolverSampler(m)


def _dir_error(sc):
    """How far the kernel's sqrt(1 - a' - sigma^2) can be from the fp64 one of the same fp32 scalars.  The kernel's radicand is
    fl(fl(1 - a') - sigma^2) (FADD then FFMA): two roundings, so it is within d = 2^-23 (|1 - a'| + sigma^2) of the exact r, and
    its square root within sqrt(max(r, 0) + d) - sqrt(max(r - d, 0)).  That is ~1e-4 at the first eta = 1 step (r = 0 up to the rounding
    of the scalars), where the square root is ill-conditioned, and negligible elsewhere.  It multiplies e_t, |e_t| <= |x| + |m|."""
    ap, sg = sc["a_prev"], sc["sigma_t"]
    r = 1.0 - ap - sg * sg
    d = EPS32 * (abs(1.0 - ap) + sg * sg)
    return math.sqrt(max(r, 0.0) + d) - math.sqrt(max(r - d, 0.0))


def _sweep(spacing, base_scale, eta, steps, three_way, guidance_rescale, worst):
    """Run both updates on every step of every S in `steps`; fold the worst error / bound per output into `worst`."""
    from viewcrafter_b200 import ops
    (x, vc, vu, vi, nz, hist), (xg, vcg, vug, vig, nzg, histg) = _inputs()
    kw_g = dict(v_uncond_img=vig, cfg_img=CFG_IMG) if three_way else {}
    kw_c = dict(v_uncond_img=vi, cfg_img=CFG_IMG) if three_way else {}
    m_mag = (vu.abs() + CFG_IMG * (vi.abs() + vu.abs()) + CFG * (vc.abs() + vi.abs()) if three_way
             else vu.abs() + CFG * (vc.abs() + vu.abs())).double()
    ddim_smp, dpm_smp = _samplers(three_way, base_scale)
    for S in steps:
        runs = []
        for (j, sd), (j2, sp) in zip(sampler_steps(ddim_smp, spacing, S, eta), sampler_steps(dpm_smp, spacing, S, eta)):
            assert j == j2 and all(sd[k] == sp[k] for k in sd), (S, j)
            guide = dict(cfg_scale=CFG, guidance_rescale=guidance_rescale)
            sd, sp = dict(sd, **guide), dict(sp, **guide)
            h = histg.clone()
            dpm = ops.dpm_update(xg, vcg, vug, nzg, sp, h, **kw_g)
            ddim = ops.ddim_update(xg, vcg, vug, nzg, sd, **kw_g)
            runs.append((j, sd, sp, ddim, dpm + (h,)))
        torch.cuda.synchronize()
        for j, sd, sp, ddim, dpm in runs:
            if sp["c_hist"] == 0.0:
                assert torch.equal(ddim[0], dpm[0]) and torch.equal(ddim[1], dpm[1]), (spacing, S, j)
            resc = max(1.0, sp["prev_scale_t"] / sp["scale_t"])
            for name, sc, got in (("ddim", sd, ddim), ("dpm", sp, dpm)):
                h_ref = hist.clone().double()
                ref = dpm_update_f64(x, vc, vu, nz, dict(sc, c_hist=sc.get("c_hist", 0.0)), h_ref, **kw_c)
                mag = (x.double().abs() + m_mag + nz.double().abs() + abs(sc.get("c_hist", 0.0)) * hist.double().abs()) * resc
                tol = 16 * EPS32 * mag
                tol_x = tol + _dir_error(sc) * (x.double().abs() + m_mag)
                for k, out in enumerate(("x_prev", "pred_x0", "x0_hist")[:len(got)]):
                    g = got[k].cpu().double()
                    r = ref[k] if k < 2 else h_ref
                    assert bool(torch.isfinite(g).all()), f"{name} {out}: non-finite output at {spacing} S={S} index {j} eta={eta}"
                    ratio = float(((g - r).abs() / (tol_x if k == 0 else tol)).max())
                    assert ratio <= 1.0, f"{name} {out}: error / bound {ratio:.3g} at {spacing} S={S} index {j} eta={eta}"
                    key = (name, out)
                    if ratio > worst.get(key, (0.0,))[0]:
                        worst[key] = (ratio, S, j)


def _report(tag, worst):
    for (name, out), (r, S, j) in sorted(worst.items()):
        print(f"{tag} {name} {out}: worst error / bound {r:.3g} (S={S}, index {j})")


@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize("base_scale", BASE_SCALES)
@pytest.mark.parametrize("spacing", SPACINGS)
def test_every_step_of_every_step_count(spacing, base_scale, eta):
    worst = {}
    _sweep(spacing, base_scale, eta, step_counts(spacing), False, 0.0, worst)
    _report(f"{spacing} base_scale={base_scale} eta={eta}:", worst)


@pytest.mark.parametrize("guidance_rescale", [0.0, 0.7])
@pytest.mark.parametrize("three_way", [False, True])
@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize("spacing", SPACINGS)
def test_guidance_grid(spacing, eta, three_way, guidance_rescale):
    for base_scale in BASE_SCALES:
        worst = {}
        _sweep(spacing, base_scale, eta, [S for S in CFG_STEPS if S in step_counts(spacing)], three_way, guidance_rescale, worst)
        _report(f"{spacing} base_scale={base_scale} eta={eta} three_way={three_way} rescale={guidance_rescale}:", worst)


@pytest.mark.parametrize("three_way", [False, True])
def test_eta_one_ddim_samplers_are_finite(three_way):
    from tests.test_dpm_solver_gpu import _ld_model, _run
    from viewcrafter_b200 import ddim, ddim_multiplecond
    model = _ld_model()
    cls = ddim_multiplecond.DDIMSampler if three_way else ddim.DDIMSampler
    for S in E2E_STEPS:
        out, inter = _run(model, cls, S, 1.0, three_way)
        bad = [k for k, t in enumerate(inter["x_inter"]) if not bool(torch.isfinite(t).all())]
        print(f"three_way={three_way} S={S}: non-finite x_inter at {bad}, output std {float(out.std()):.3g}")
        assert not bad and all(bool(torch.isfinite(t).all()) for t in [out] + inter["pred_x0"]), (S, bad)


@pytest.mark.parametrize("three_way", [False, True])
def test_eta_one_four_steps_vs_oracle(three_way):
    """S = 4, eta = 1, CFG 7.5 (cfg_img 2.0), rescale 0.7: the loop of test_ddim_sample_three_steps_vs_oracle one step longer, where the
    first step's fused radicand is below zero and the reference's is exactly zero."""
    from oracle import lvdm_oracle as O
    from oracle import synth
    from viewcrafter_b200 import ddim, ddim_multiplecond
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.7)
    unet = model.model.diffusion_model
    sd = synth.synth_state_dict(synth.module_shapes(unet), seed=41)
    unet.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    g = torch.Generator().manual_seed(42)
    T, H, W, S = 5, 8, 8, 4
    shape = (1, 4, T, H, W)
    x_T, cc = torch.randn(shape, generator=g), torch.randn(shape, generator=g)
    ctx_c, ctx_u, ctx_i = (torch.randn(1, 333, 1024, generator=g) for _ in range(3))
    fs = torch.tensor([10])
    c, uc, ui = ({"c_crossattn": [k.cuda()], "c_concat": [cc.cuda()]} for k in (ctx_c, ctx_u, ctx_i))
    kw = dict(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui) if three_way else {}
    sampler = (ddim_multiplecond.DDIMSampler if three_way else ddim.DDIMSampler)(model, batch_cfg=True)
    torch.manual_seed(43)
    out, inter = sampler.sample(S=S, batch_size=1, shape=shape[1:], conditioning=c, eta=1.0, verbose=False, x_T=x_T.cuda(),
                                unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=fs.cuda(),
                                timestep_spacing="uniform_trailing", guidance_rescale=0.7, **kw)
    torch.manual_seed(43)
    noises = [torch.randn(shape, device="cuda").cpu() for _ in range(S)]
    sched = O.model_schedule(base_scale=0.7)

    def model_fn(x, t, cond):
        with torch.no_grad():
            return O.unet_forward(sd, torch.cat([x, cc], 1), t, cond, fs)

    extra = dict(fixed_prev_scale=False, uncond_img=ctx_i, cfg_img=2.0) if three_way else {}
    ref, ref_inter = O.ddim_sample(model_fn, sched, shape, S, ctx_c, ctx_u, x_T, noises, **extra)
    assert bool(torch.isfinite(ref).all())
    err = (out.cpu() - ref).abs()
    print(f"three_way={three_way} ddim S=4 eta=1: max err {float(err.max()):.4g} mean {float(err.mean()):.4g} ref std {float(ref.std()):.3g}")
    assert len(inter["x_inter"]) == len(ref_inter["x_inter"])
    assert float(err.max()) <= 0.15 and float(err.mean()) <= 0.02 and math.isfinite(float(err.max()))
