"""DPM-Solver++(3M) SDE on the GPU (vc_dpm3_update, viewcrafter_b200.dpm_solver.DPMSolver3MSDESampler):
  * the fused update against the fp64 restatement of tests/test_dpm3_solver_cpu.py on random tensors, over two- and three-way guidance,
    guidance rescale, dynamic rescale and (c1, c2) zero / non-zero; c2 = 0 is ops.dpm_update and c1 = c2 = 0 ops.ddim_update bit for bit;
  * with the model_channels=64 U-Net, uniform_trailing runs of S <= 4 and the first three steps of S = 10 are torch.equal to the 2M
    sampler with the same seed (two- and three-way guidance);
  * the analytic Gaussian SDE ordering of the CPU test with the real kernel;
  * reproducible mode: batch_cfg on / off, B=2 against its rows, eager against graph replay, and replica groups R=2 / R=4 run in one
    process against the sequential image_guided_synthesis call (outputs and generator end states torch.equal)."""
import math

import pytest
import torch

from tests.test_dpm3_solver_cpu import dpm3_update_f64
from tests.test_dpm_solver_cpu import S0, GaussianModel, _alphas
from tests.test_dpm_solver_gpu import _ld_model, _run, _scalars, reproducible  # noqa: F401  (reproducible: a fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
EPS32 = 2.0 ** -23


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _scalars3(dynamic, c1, c2, guidance_rescale):
    sc = _scalars(1.0, dynamic, 0.0, guidance_rescale)
    del sc["c_hist"]
    f = lambda v: float(torch.tensor(v, dtype=torch.float32))
    return dict(sc, c1=f(c1), c2=f(c2))


@pytest.mark.parametrize("three_way", [False, True])
@pytest.mark.parametrize("guidance_rescale", [0.0, 0.7])
@pytest.mark.parametrize("dynamic", [False, True])
def test_update_matches_fp64_restatement(three_way, guidance_rescale, dynamic):
    from viewcrafter_b200 import ops
    g = torch.Generator().manual_seed(2)
    n = 4 * 5 * 40 * 64 + 3
    x, vc, vu, vi, nz, h1, h2 = (torch.randn(n, generator=g) * s for s in (1.0, 1.0, 1.2, 1.1, 1.0, 0.9, 0.8))
    kw = dict(v_uncond_img=vi.cuda(), cfg_img=2.0) if three_way else {}
    for c1, c2 in ((0.0, 0.0), (0.173, 0.0), (0.173, -0.061), (0.0, -0.061)):
        sc = _scalars3(dynamic, c1, c2, guidance_rescale)
        h1_gpu, h2_gpu = h1.cuda(), h2.cuda()
        xp, p0 = ops.dpm3_update(x.cuda(), vc.cuda(), vu.cuda(), nz.cuda(), sc, h1_gpu, h2_gpu, **kw)
        h2_ref = h2.clone().double()
        xp_ref, p0_ref = dpm3_update_f64(x, vc, vu, nz, sc, h1, h2_ref, **({"v_uncond_img": vi, "cfg_img": 2.0} if three_way else {}))
        # magnitude of the terms each output sums (the guidance combine dominates at cfg 7.5)
        m_mag = vu.abs() + 2.0 * (vi.abs() + vu.abs()) + 7.5 * (vc.abs() + vi.abs()) if three_way else vu.abs() + 7.5 * (vc.abs() + vu.abs())
        mag = (x.double().abs() + m_mag.double() + nz.double().abs() + abs(c1) * h1.double().abs()
               + abs(c2) * (h1.double().abs() + h2.double().abs()))
        tol = 16 * EPS32 * mag
        assert torch.equal(h1_gpu.cpu(), h1)                           # only read
        for name, got, ref in (("x_prev", xp, xp_ref), ("pred_x0", p0, p0_ref), ("x0_hist2", h2_gpu, h2_ref)):
            err = (got.cpu().double() - ref).abs()
            print(f"three_way={three_way} rescale={guidance_rescale} dynamic={dynamic} c1={c1} c2={c2}: {name} max err "
                  f"{float(err.max()):.3g}, max err / bound {float((err / tol).max()):.3g}")
            assert bool((err <= tol).all()), name
        if c2 == 0.0:
            h = h1.cuda()
            xd, pd = ops.dpm_update(x.cuda(), vc.cuda(), vu.cuda(), nz.cuda(), dict(sc, c_hist=sc["c1"]), h, **kw)
            assert torch.equal(xd, xp) and torch.equal(pd, p0) and torch.equal(h, h2_gpu)
        if c1 == 0.0 and c2 == 0.0:
            xd, pd = ops.ddim_update(x.cuda(), vc.cuda(), vu.cuda(), nz.cuda(), sc, **kw)
            assert torch.equal(xd, xp) and torch.equal(pd, p0)


def test_update_rejects_bad_arguments():
    from viewcrafter_b200 import _lib, ops
    x = torch.randn(64, device="cuda")
    for c1, c2 in ((0.5, float("nan")), (float("inf"), 0.0)):
        with pytest.raises(_lib.VcError, match="finite"):
            ops.dpm3_update(x, x.clone(), None, x.clone(), _scalars3(False, c1, c2, 0.0), torch.zeros_like(x), torch.zeros_like(x))
    sc = _scalars3(False, 0.5, 0.25, 0.0)
    h = torch.zeros_like(x)
    with pytest.raises(_lib.VcError, match="alias"):
        ops.dpm3_update(x, x.clone(), None, x.clone(), sc, h, h)
    with pytest.raises(_lib.VcError, match="alias"):
        ops.dpm3_update(h, x.clone(), None, x.clone(), sc, torch.zeros_like(x), h)


def _classes(three_way):
    from viewcrafter_b200 import dpm_solver
    if three_way:
        return dpm_solver.DPMSolverSamplerMultiCond, dpm_solver.DPMSolver3MSDESamplerMultiCond
    return dpm_solver.DPMSolverSampler, dpm_solver.DPMSolver3MSDESampler


@pytest.mark.parametrize("three_way", [False, True])
def test_first_three_steps_are_the_2m_steps_bit_for_bit(three_way):
    model = _ld_model()
    cls2, cls3 = _classes(three_way)
    for S in (1, 2, 3, 4, 10):
        (a, ia), (b, ib) = (_run(model, cls, S, 1.0, three_way) for cls in (cls2, cls3))
        if S <= 4:
            assert torch.equal(a, b) and torch.equal(ia["pred_x0"][-1], ib["pred_x0"][-1]), S
        else:
            for k in (1, 2, 3):                  # after the first, second and third step
                assert torch.equal(ia["x_inter"][k], ib["x_inter"][k]) and torch.equal(ia["pred_x0"][k], ib["pred_x0"][k]), k
            d = float((a - b).abs().max())
            print(f"three_way={three_way} S=10: 3M vs 2M output max |diff| {d:.3g}")
            assert d > 0 and math.isfinite(d)


def test_gaussian_sde_ordering_with_the_kernel():
    """eta = 1 on the Gaussian problem with the real kernels: the error of the output's std over 4e5 samples, with the same x_T and
    noise seeds for every solver at each S."""
    from viewcrafter_b200.ddim import DDIMSampler
    from viewcrafter_b200.dpm_solver import DPMSolver3MSDESampler, DPMSolverSampler
    ac = _alphas()
    model = GaussianModel()
    for k in ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod"):
        setattr(model, k, getattr(model, k).cuda())
    n = 400_000
    std_exact = math.sqrt(ac[0] * S0 * S0 + 1 - ac[0])
    errs = {}
    for S in (10, 15, 20, 50):
        for k, cls in enumerate((DDIMSampler, DPMSolverSampler, DPMSolver3MSDESampler)):
            x_T = torch.randn(1, 1, 1, n, generator=torch.Generator().manual_seed(S)).cuda()
            torch.manual_seed(100 + S)
            out, _ = cls(model).sample(S=S, batch_size=1, shape=(1, 1, n), x_T=x_T, eta=1.0, verbose=False,
                                       timestep_spacing="uniform_trailing")
            errs[S, k] = float(out.double().std()) - std_exact
        print(f"S={S}: std error DDIM {errs[S, 0]:+.4f}, 2M SDE {errs[S, 1]:+.4f}, 3M SDE {errs[S, 2]:+.4f}")
    for S in (10, 15, 20):
        assert abs(errs[S, 2]) < abs(errs[S, 1]), S
    assert abs(errs[10, 2]) < abs(errs[50, 0])


@pytest.mark.parametrize("three_way", [False, True])
def test_reproducible_batching_and_graph_replay(three_way, reproducible):  # noqa: F811
    _, cls3 = _classes(three_way)
    model = _ld_model()
    unet = model.model.diffusion_model
    eager, _ = _run(model, cls3, 6, 1.0, three_way, batch_cfg=True)
    unet.enable_cuda_graph()
    graph, _ = _run(model, cls3, 6, 1.0, three_way, batch_cfg=True)
    assert unet.graph_replayed_launches > 0
    unbatched, _ = _run(model, cls3, 6, 1.0, three_way, batch_cfg=False)
    for name, y in (("graph replay", graph), ("batch_cfg off", unbatched)):
        print(f"three_way={three_way}: eager vs {name}: max |diff| {float((eager - y).abs().max()):.3g}")
        assert torch.equal(eager, y), name
    b2, _ = _run(model, cls3, 6, 1.0, three_way, B=2)
    for b in range(2):
        b1, _ = _run(model, cls3, 6, 1.0, three_way, B=2, rows=(b, b + 1))
        print(f"three_way={three_way}: B=2 row {b} vs B=1: max |diff| {float((b2[b:b + 1] - b1).abs().max()):.3g}")
        assert torch.equal(b2[b:b + 1], b1), b


@pytest.mark.parametrize("three_way", [False, True])
def test_replica_groups_match_the_sequential_call(three_way, reproducible):  # noqa: F811
    from tests.test_replicas_gpu import _model, _one_process_replicas
    from viewcrafter_b200.synthesis import image_guided_synthesis
    T, H, W = 5, 40, 64
    model = _model(64)
    B, n = 2, 2
    videos = (torch.rand(B, 3, T, 8 * H, 8 * W, generator=torch.Generator().manual_seed(94)) * 2 - 1).cuda()
    kw = dict(n_samples=n, ddim_steps=6, ddim_eta=1.0, unconditional_guidance_scale=7.5, cfg_img=(2.0 if three_way else None), fs=10,
              text_input=True, multiple_cond_cfg=three_way, timestep_spacing="uniform_trailing", guidance_rescale=0.7, condition_index=[0],
              sampler="dpmpp_3m_sde")

    def run():
        torch.manual_seed(95)
        out = image_guided_synthesis(model, ["a photo"] * B, videos, [B, 4, T, H, W], **kw)
        torch.cuda.synchronize()
        return out, torch.cuda.get_rng_state(), torch.get_rng_state()

    ref, cuda_rng, cpu_rng = run()
    torch.manual_seed(95)
    out_2m = image_guided_synthesis(model, ["a photo"] * B, videos, [B, 4, T, H, W], **dict(kw, sampler="dpmpp_2m"))
    assert bool(torch.isfinite(ref).all()) and bool(torch.isfinite(out_2m).all())
    assert not torch.equal(out_2m, ref)                  # S = 6 has two third-order steps
    for R in (2, 4):
        store = {}
        for g in range(R):
            model._replicas = _one_process_replicas(g, R, store)
            out, c_rng, p_rng = run()
            assert torch.equal(c_rng, cuda_rng) and torch.equal(p_rng, cpu_rng), (R, g)
        del model._replicas
        print(f"three_way={three_way} R={R}: every group's jobs vs the sequential call: max |diff| {float((out - ref).abs().max()):.3g}")
        assert out.shape == ref.shape and torch.equal(out, ref), R
