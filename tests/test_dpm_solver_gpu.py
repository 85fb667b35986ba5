"""DPM-Solver++(2M) on the GPU (vc_dpm_update, viewcrafter_b200.dpm_solver):
  * the fused update against the fp64 restatement of tests/test_dpm_solver_cpu.py on random tensors, over two- and three-way guidance,
    guidance rescale, dynamic rescale, eta 0 / 1 and c_hist zero / non-zero; c_hist = 0 is ops.ddim_update bit for bit;
  * with the model_channels=64 U-Net, runs whose steps are all first order, and the first two steps of S = 10, are torch.equal to
    DDIMSampler with the same seed and eta (two- and three-way guidance);
  * the analytic Gaussian convergence of the CPU test with the real kernel;
  * reproducible mode: batch_cfg on / off, B=2 against B=1, eager against graph replay, and replica groups R=2 / R=4 run in one process
    against the sequential image_guided_synthesis call (outputs and generator end states torch.equal)."""
import math

import pytest
import torch

from tests.test_dpm_solver_cpu import MU, ODE_TABLE, GaussianModel, S0, _alphas, _solve_ref, dpm_update_f64

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
EPS32 = 2.0 ** -23


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.fixture
def reproducible():
    from viewcrafter_b200 import set_reproducible
    prev = set_reproducible(True)
    yield
    set_reproducible(prev)


def _scalars(eta, dynamic, c_hist, guidance_rescale):
    a, a_prev = 0.35, 0.55
    sigma = eta * math.sqrt((1 - a_prev) / (1 - a) * (1 - a / a_prev))
    f = lambda v: float(torch.tensor(v, dtype=torch.float32))
    return dict(cfg_scale=7.5, guidance_rescale=guidance_rescale, sqrt_ac_t=f(math.sqrt(a)), sqrt_1mac_t=f(math.sqrt(1 - a)),
                a_prev=f(a_prev), sigma_t=f(sigma), scale_t=f(0.7 if dynamic else 1.0), prev_scale_t=f(0.74 if dynamic else 1.0),
                c_hist=f(c_hist))


@pytest.mark.parametrize("three_way", [False, True])
@pytest.mark.parametrize("guidance_rescale", [0.0, 0.7])
@pytest.mark.parametrize("dynamic", [False, True])
@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_update_matches_fp64_restatement(three_way, guidance_rescale, dynamic, eta):
    from viewcrafter_b200 import ops
    g = torch.Generator().manual_seed(1)
    n = 4 * 5 * 40 * 64 + 3
    x, vc, vu, vi, nz, hist = (torch.randn(n, generator=g) * s for s in (1.0, 1.0, 1.2, 1.1, 1.0, 0.9))
    for c_hist in (0.0, 0.173):
        sc = _scalars(eta, dynamic, c_hist, guidance_rescale)
        kw = dict(v_uncond_img=vi.cuda(), cfg_img=2.0) if three_way else {}
        h_gpu = hist.cuda()
        xp, p0 = ops.dpm_update(x.cuda(), vc.cuda(), vu.cuda(), nz.cuda(), sc, h_gpu, **kw)
        h_ref = hist.clone().double()
        xp_ref, p0_ref = dpm_update_f64(x, vc, vu, nz, sc, h_ref, **({"v_uncond_img": vi, "cfg_img": 2.0} if three_way else {}))
        # magnitude of the terms each output sums (the guidance combine dominates at cfg 7.5)
        m_mag = vu.abs() + 2.0 * (vi.abs() + vu.abs()) + 7.5 * (vc.abs() + vi.abs()) if three_way else vu.abs() + 7.5 * (vc.abs() + vu.abs())
        mag = x.double().abs() + m_mag.double() + nz.double().abs() + abs(c_hist) * hist.double().abs()
        tol = 16 * EPS32 * mag
        for name, got, ref in (("x_prev", xp, xp_ref), ("pred_x0", p0, p0_ref), ("x0_hist", h_gpu, h_ref)):
            err = (got.cpu().double() - ref).abs()
            print(f"three_way={three_way} rescale={guidance_rescale} dynamic={dynamic} eta={eta} c={c_hist}: {name} max err "
                  f"{float(err.max()):.3g}, max err / bound {float((err / tol).max()):.3g}")
            assert bool((err <= tol).all()), name
        if c_hist == 0.0:
            xd, pd = ops.ddim_update(x.cuda(), vc.cuda(), vu.cuda(), nz.cuda(), sc, **kw)
            assert torch.equal(xd, xp) and torch.equal(pd, p0)


def test_update_rejects_bad_arguments():
    from viewcrafter_b200 import _lib, ops
    x = torch.randn(64, device="cuda")
    sc = _scalars(0.0, False, float("nan"), 0.0)
    with pytest.raises(_lib.VcError, match="c_hist"):
        ops.dpm_update(x, x.clone(), None, x.clone(), sc, torch.zeros_like(x))
    sc["c_hist"] = 0.5
    with pytest.raises(_lib.VcError, match="alias"):
        h = torch.zeros_like(x)
        ops.dpm_update(h, x, None, x, sc, h)


def _ld_model(seed=41):
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.7)
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), seed=seed), strict=True)
    return model.cuda().eval()


def _conds(B=1, seed=42, shape=(4, 5, 40, 64)):
    g = torch.Generator().manual_seed(seed)
    x_T, cc = torch.randn(B, *shape, generator=g).cuda(), torch.randn(B, *shape, generator=g).cuda()
    c, uc, ui = ({"c_crossattn": [torch.randn(B, 333, 1024, generator=g).cuda()], "c_concat": [cc]} for _ in range(3))
    return x_T, c, uc, ui


def _run(model, cls, S, eta, three_way, batch_cfg=True, B=1, x_T=None, rows=None, seed=43, guidance_rescale=0.7):
    xT, c, uc, ui = _conds(B)
    kw = dict(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui) if three_way else {}
    if rows is not None:
        sl = lambda d: {k: [t[rows[0]:rows[1]] for t in v] for k, v in d.items()}
        c, uc = sl(c), sl(uc)
        if three_way:
            kw["unconditional_conditioning_img_nonetext"] = sl(ui)
        kw["_rng_rows"] = rows
    torch.manual_seed(seed)
    out, inter = cls(model, batch_cfg=batch_cfg).sample(
        S=S, batch_size=B, shape=xT.shape[1:], conditioning=c, eta=eta, verbose=False, x_T=x_T, log_every_t=1,
        unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=torch.tensor([10] * (B if rows is None else 1)).cuda(),
        timestep_spacing="uniform_trailing", guidance_rescale=guidance_rescale, **kw)
    return out, inter


def _classes(three_way):
    from viewcrafter_b200 import ddim, ddim_multiplecond, dpm_solver
    if three_way:
        return ddim_multiplecond.DDIMSampler, dpm_solver.DPMSolverSamplerMultiCond
    return ddim.DDIMSampler, dpm_solver.DPMSolverSampler


@pytest.mark.parametrize("three_way", [False, True])
def test_first_order_steps_are_ddim_bit_for_bit(three_way):
    model = _ld_model()
    ddim_cls, dpm_cls = _classes(three_way)
    for eta in (0.0, 1.0):
        for S in (1, 2, 10):
            (a, ia), (b, ib) = (_run(model, cls, S, eta, three_way) for cls in (ddim_cls, dpm_cls))
            if S < 10:
                assert torch.equal(a, b) and torch.equal(ia["pred_x0"][-1], ib["pred_x0"][-1]), (S, eta)
            else:
                for k in (1, 2):                 # after the first and the second step
                    assert torch.equal(ia["x_inter"][k], ib["x_inter"][k]) and torch.equal(ia["pred_x0"][k], ib["pred_x0"][k]), (k, eta)
                d = float((a - b).abs().max())
                print(f"three_way={three_way} eta={eta} S=10: DPM vs DDIM output max |diff| {d:.3g}")
                assert d > 0 and math.isfinite(d)


def test_four_step_sde_is_finite():
    """eta = 1, 4 uniform_trailing steps: 1 - a' - sigma^2 of the first step's fp32 scalars rounds below 0; the update clamps it."""
    from viewcrafter_b200 import dpm_solver
    from viewcrafter_b200.schedule import ddim_timesteps
    model = _ld_model()
    smp = dpm_solver.DPMSolverSampler(model)
    smp.make_schedule(4, "uniform_trailing", 1.0, verbose=False)
    sc = smp.step_scalars(3, int(ddim_timesteps("uniform_trailing", 4, 1000)[3]))
    print(f"first step: 1 - a' - sigma^2 = {1.0 - sc['a_prev'] - sc['sigma_t'] ** 2:.3g} (fp64 of the fp32 scalars)")
    out, inter = _run(model, dpm_solver.DPMSolverSampler, 4, 1.0, False)
    assert all(bool(torch.isfinite(t).all()) for t in [out] + inter["x_inter"] + inter["pred_x0"])


def test_gaussian_convergence_with_the_kernel():
    from viewcrafter_b200.ddim import DDIMSampler
    from viewcrafter_b200.dpm_solver import DPMSolverSampler
    ac = _alphas()
    model = GaussianModel()
    for k in ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod"):
        setattr(model, k, getattr(model, k).cuda())
    x_T = torch.linspace(-3, 3, 101, dtype=torch.float64).reshape(1, 1, 1, 101)
    exact = math.sqrt(ac[0]) * MU + math.sqrt(ac[0] * S0 * S0 + 1 - ac[0]) * x_T
    errs = {}
    for S, tabs in ODE_TABLE.items():
        for k, cls in enumerate((DDIMSampler, DPMSolverSampler)):
            out, _ = cls(model).sample(S=S, batch_size=1, shape=(1, 1, 101), x_T=x_T.float().cuda(), eta=0.0, verbose=False,
                                       timestep_spacing="uniform_trailing")
            out = out.cpu().double()
            ref = _solve_ref(ac, S, k == 1, x_T.float().double())
            d = float((out - ref).abs().max())
            errs[S, k] = float((out - exact).abs().max())
            print(f"S={S} {cls.__name__}: max error {errs[S, k]:.6f} (table {tabs[k]}), kernel vs fp64 restatement {d:.2e}")
            assert d < 1e-5 * float(ref.abs().max())
            assert abs(errs[S, k] - float(tabs[k])) <= 0.5 * 10.0 ** -len(tabs[k].split(".")[1])
    assert all(errs[S, 1] < errs[S, 0] for S in ODE_TABLE) and errs[20, 1] < errs[50, 0]


@pytest.mark.parametrize("three_way", [False, True])
def test_reproducible_batching_and_graph_replay(three_way, reproducible):
    _, dpm_cls = _classes(three_way)
    model = _ld_model()
    unet = model.model.diffusion_model
    eager, _ = _run(model, dpm_cls, 5, 1.0, three_way, batch_cfg=True)
    unet.enable_cuda_graph()
    graph, _ = _run(model, dpm_cls, 5, 1.0, three_way, batch_cfg=True)
    assert unet.graph_replayed_launches > 0
    unbatched, _ = _run(model, dpm_cls, 5, 1.0, three_way, batch_cfg=False)
    for name, y in (("graph replay", graph), ("batch_cfg off", unbatched)):
        print(f"three_way={three_way}: eager vs {name}: max |diff| {float((eager - y).abs().max()):.3g}")
        assert torch.equal(eager, y), name
    b2, _ = _run(model, dpm_cls, 5, 1.0, three_way, B=2)
    for b in range(2):
        b1, _ = _run(model, dpm_cls, 5, 1.0, three_way, B=2, rows=(b, b + 1))
        print(f"three_way={three_way}: B=2 row {b} vs B=1: max |diff| {float((b2[b:b + 1] - b1).abs().max()):.3g}")
        assert torch.equal(b2[b:b + 1], b1), b


@pytest.mark.parametrize("three_way", [False, True])
def test_replica_groups_match_the_sequential_call(three_way, reproducible):
    from tests.test_replicas_gpu import _model, _one_process_replicas
    from viewcrafter_b200.synthesis import image_guided_synthesis
    T, H, W = 5, 40, 64
    model = _model(64)
    B, n = 2, 2
    videos = (torch.rand(B, 3, T, 8 * H, 8 * W, generator=torch.Generator().manual_seed(94)) * 2 - 1).cuda()
    kw = dict(n_samples=n, ddim_steps=5, ddim_eta=1.0, unconditional_guidance_scale=7.5, cfg_img=(2.0 if three_way else None), fs=10,
              text_input=True, multiple_cond_cfg=three_way, timestep_spacing="uniform_trailing", guidance_rescale=0.7, condition_index=[0],
              sampler="dpmpp_2m")

    def run():
        torch.manual_seed(95)
        out = image_guided_synthesis(model, ["a photo"] * B, videos, [B, 4, T, H, W], **kw)
        torch.cuda.synchronize()
        return out, torch.cuda.get_rng_state(), torch.get_rng_state()

    ref, cuda_rng, cpu_rng = run()
    ddim_out = image_guided_synthesis(model, ["a photo"] * B, videos, [B, 4, T, H, W], **dict(kw, sampler="ddim"))
    assert bool(torch.isfinite(ref).all()) and bool(torch.isfinite(ddim_out).all())
    assert not torch.equal(ddim_out, ref)                # S = 5 has two second-order steps
    for R in (2, 4):
        store = {}
        for g in range(R):
            model._replicas = _one_process_replicas(g, R, store)
            out, c_rng, p_rng = run()
            assert torch.equal(c_rng, cuda_rng) and torch.equal(p_rng, cpu_rng), (R, g)
        del model._replicas
        print(f"three_way={three_way} R={R}: every group's jobs vs the sequential call: max |diff| {float((out - ref).abs().max()):.3g}")
        assert out.shape == ref.shape and torch.equal(out, ref), R
