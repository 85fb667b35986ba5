"""DPM-Solver++(3M) SDE sampler (viewcrafter_b200.dpm_solver.DPMSolver3MSDESampler) on the CPU:
  * the host coefficients (schedule.dpm3_coefficients) against an independent fp64 restatement in alpha / sigma form that evaluates
    k-diffusion's phi2 d1 - phi3 d2 on unit differences, for every spacing, and the fallbacks to first order and to the 2M step;
  * the sampler loop on the analytic Gaussian problem of tests/test_dpm_solver_cpu.py at eta = 1, with ops.dpm3_update replaced by the
    fp64 restatement below (dpm3_update_f64, also the GPU test's reference): against an independent loop, and the std error of
    DDIM, 2M SDE and 3M SDE over 4e5 samples (the table of INTEGRATION.md "Samplers" is this test's printed output);
  * the options and the eta the sampler rejects, before any forward, also from image_guided_synthesis."""
import math

import numpy as np
import pytest
import torch

from tests.test_dpm_solver_cpu import MU, S0, SPACINGS, GaussianModel, _alphas, ddim_update_f64, dpm_update_f64, lam
from viewcrafter_b200 import ops, schedule
from viewcrafter_b200.ddim import DDIMSampler
from viewcrafter_b200.dpm_solver import (DPMSolver3MSDESampler, DPMSolver3MSDESamplerMultiCond, DPMSolverSampler,
                                         DPMSolverSamplerMultiCond)

# std error of the output at eta = 1: the step counts printed for the table of INTEGRATION.md
TABLE_STEPS = (8, 10, 12, 15, 20, 25, 50)


def dpm3_update_f64(x, v_cond, v_uncond, noise, sc, x0_hist1, x0_hist2, v_uncond_img=None, cfg_img=0.0):
    """fp64 restatement of ops.dpm3_update: dpm_update_f64 with c_hist = c1, plus c2 (x0_hist1 - x0_hist2).  Writes this step's x0 into
    x0_hist2 and returns fp64 (x_prev, pred_x0)."""
    m1 = x0_hist1.double()
    x0 = m1.clone()                  # dpm_update_f64 reads its history only when c_hist != 0, then overwrites it with this step's x0
    x_prev, p0 = dpm_update_f64(x, v_cond, v_uncond, noise, dict(sc, c_hist=sc["c1"]), x0, v_uncond_img, cfg_img)
    if sc["c2"] != 0.0:
        x_prev = x_prev + sc["c2"] * (m1 - x0_hist2.double())
    x0_hist2.copy_(x0)
    return x_prev, p0


def coefficients_ref(ac, ts):
    """(c1, c2) of every step, restated from the definitions with alpha and sigma: the 3M step evaluates k-diffusion's
    x += alpha' (phi2 d1 - phi3 d2) on (m0, m1, m2) = (1, 0, 0) and (1, 1, 0), i.e. on unit differences m0 - m1 and m1 - m2."""
    ts = [int(t) for t in ts[::-1]]
    S = len(ts)
    nxt = lambda i: ac[ts[i + 1]] if i + 1 < S else ac[0]
    hs = [lam(nxt(i)) - lam(ac[t]) for i, t in enumerate(ts)]
    c1, c2 = np.zeros(S), np.zeros(S)
    for i, t in enumerate(ts):
        a, an = ac[t], nxt(i)
        h = hs[i]
        if i == 0 or i == S - 1 or not math.isfinite(hs[i - 1]) or h == 0.0 or hs[i - 1] == 0.0:
            continue
        ratio = (math.sqrt(1 - an) / math.sqrt(1 - a)) * (math.sqrt(a) / math.sqrt(an))       # exp(-h)
        r0 = hs[i - 1] / h
        if i < 2 or not math.isfinite(hs[i - 2]) or hs[i - 2] == 0.0:
            c1[i] = math.sqrt(an) * (1.0 - ratio ** 2) / (2.0 * r0)                            # the 2M SDE step
            continue
        r1 = hs[i - 2] / h
        he = 2.0 * h
        phi2 = 1.0 - (1.0 - ratio ** 2) / he
        phi3 = phi2 / he - 0.5

        def step(m0, m1, m2):
            d1_0, d1_1 = (m0 - m1) / r0, (m1 - m2) / r1
            d1 = d1_0 + (d1_0 - d1_1) * r0 / (r0 + r1)
            d2 = (d1_0 - d1_1) / (r0 + r1)
            return math.sqrt(an) * (phi2 * d1 - phi3 * d2)
        c1[i], c2[i] = step(1.0, 0.0, 0.0), step(1.0, 1.0, 0.0)
    return c1[::-1], c2[::-1]                      # DDIM index order


@pytest.mark.parametrize("spacing", SPACINGS)
def test_coefficients_match_the_alpha_sigma_restatement(spacing):
    ac = _alphas()
    for S in (1, 2, 3, 4, 5, 10, 25, 50):
        ts = schedule.ddim_timesteps(spacing, S, 1000)
        if ts.max() >= 1000:                 # "uniform" at S = 3 reaches t = 1000: DDIM's own tables fail there (the reference's too)
            with pytest.raises(IndexError):
                schedule.dpm3_coefficients(ac, ts)
            continue
        S = len(ts)
        c1, c2 = schedule.dpm3_coefficients(ac, ts)
        r1, r2 = coefficients_ref(ac, ts)
        for c in (c1, c2):
            assert c.shape == (S,) and c.dtype == np.float64 and np.all(np.isfinite(c)), (spacing, S)
        assert np.array_equal(c1 == 0, r1 == 0) and np.array_equal(c2 == 0, r2 == 0), (spacing, S, c1, c2, r1, r2)
        # phi3 = phi2 / h_e - 1/2 cancels to about h_e / 6, so the restatement's (1 - e^{-h_e}) / h_e form loses a few digits
        np.testing.assert_allclose(c1, r1, rtol=1e-9, atol=0, err_msg=f"c1 {spacing} S={S}")
        np.testing.assert_allclose(c2, r2, rtol=1e-9, atol=0, err_msg=f"c2 {spacing} S={S}")


@pytest.mark.parametrize("spacing", SPACINGS)
def test_fallbacks(spacing):
    """c1 = c2 = 0 exactly where the 2M c is 0; c2 = 0 and c1 the 2M c bit for bit where x0_{i-2} is not usable."""
    ac = _alphas()
    for S in (1, 2, 3, 4, 5, 10, 25, 50):
        ts = schedule.ddim_timesteps(spacing, S, 1000)
        if ts.max() >= 1000:
            continue
        S = len(ts)
        c1, c2 = schedule.dpm3_coefficients(ac, ts)
        c = schedule.dpm_coefficients(ac, ts, 1.0)
        assert np.array_equal(c1 == 0, c == 0) and np.all(c2[c == 0] == 0), (spacing, S)
        assert np.array_equal(c1[c2 == 0], c[c2 == 0]), (spacing, S)
        if spacing != "quad" and S >= 3:
            # sampling step i is DDIM index S - 1 - i; the first step, the last, and under zero-terminal SNR the step after the a = 0 one
            # are first order, and the next step (x0_{i-2} from the a = 0 step, or absent) is the 2M step
            zero_start = ac[ts[-1]] == 0
            first_order = {S - 1, 0} | ({S - 2} if zero_start else set())
            second_order = ({S - 3} if zero_start else {S - 2}) - {0}
            assert {j for j in range(S) if c1[j] == 0} == first_order, (spacing, S, c1)
            assert {j for j in range(S) if c2[j] == 0} == first_order | second_order, (spacing, S, c2)
    if spacing == "uniform_trailing":
        c1, c2 = schedule.dpm3_coefficients(ac, schedule.ddim_timesteps(spacing, 10, 1000))
        assert np.all(c1[1:7] > 0) and np.all(c2[1:7] < 0) and c2[7] == 0 and c1[7] > 0


def _solve_3m(ac, S, x, noises):
    """Independent fp64 restatement of DPM-Solver++(3M) SDE (eta = 1) on the Gaussian problem: the DDIM eta = 1 step plus k-diffusion's
    phi2 d1 - phi3 d2 (or the 2M SDE correction), with the first-order and 2M fallbacks.  The latent and the x0 history are held in fp32
    between steps, as the sampler holds them."""
    ts = [int(t) for t in schedule.ddim_timesteps("uniform_trailing", S, 1000)[::-1]]
    ms, hs = [], []
    for i, t in enumerate(ts):
        x = x.float().double()
        a, an = ac[t], (ac[ts[i + 1]] if i + 1 < S else ac[0])
        x0 = MU + math.sqrt(a) * S0 * S0 / (a * S0 * S0 + 1 - a) * (x - math.sqrt(a) * MU)
        eps = (x - math.sqrt(a) * x0) / math.sqrt(1 - a)
        sig = math.sqrt((1 - an) / (1 - a) * (1 - a / an))
        xn = math.sqrt(an) * x0 + math.sqrt(max(1 - an - sig * sig, 0.0)) * eps + sig * noises[i]
        h = lam(an) - lam(a)
        if 0 < i < S - 1 and math.isfinite(hs[-1]) and h != 0 and hs[-1] != 0:
            he, r0 = 2 * h, hs[-1] / h
            if i >= 2 and math.isfinite(hs[-2]) and hs[-2] != 0:
                r1 = hs[-2] / h
                d1_0, d1_1 = (x0 - ms[-1]) / r0, (ms[-1] - ms[-2]) / r1
                d1 = d1_0 + (d1_0 - d1_1) * r0 / (r0 + r1)
                d2 = (d1_0 - d1_1) / (r0 + r1)
                phi2 = math.expm1(-he) / he + 1
                xn = xn + math.sqrt(an) * (phi2 * d1 - (phi2 / he - 0.5) * d2)
            else:
                xn = xn + math.sqrt(an) * -math.expm1(-he) / (2 * r0) * (x0 - ms[-1])
        ms.append(x0.float().double())
        hs.append(h)
        x = xn
    return x


def _patch(monkeypatch):
    monkeypatch.setattr(ops, "dpm3_update", dpm3_update_f64)
    monkeypatch.setattr(ops, "dpm_update", dpm_update_f64)
    monkeypatch.setattr(ops, "ddim_update", ddim_update_f64)


def _sample(cls, S, x_T, monkeypatch, seed):
    _patch(monkeypatch)
    model = GaussianModel()
    torch.manual_seed(seed)
    kw = dict(unconditional_conditioning_img_nonetext=None) if cls in (DPMSolverSamplerMultiCond, DPMSolver3MSDESamplerMultiCond) else {}
    out, inter = cls(model).sample(S=S, batch_size=1, shape=tuple(x_T.shape[1:]), x_T=x_T, eta=1.0, verbose=False, log_every_t=1,
                                   timestep_spacing="uniform_trailing", **kw)
    return out.double(), inter, model


def test_sampler_matches_the_independent_loop(monkeypatch):
    """eta = 1 with the draws the sampler makes (x_T, then one noise tensor per step, like DDIMSampler.sample)."""
    ac = _alphas()
    for S in (4, 5, 10, 25):
        n = 64
        torch.manual_seed(7)
        draws = [torch.randn(1, 1, 1, n) for _ in range(S + 1)]
        _patch(monkeypatch)
        model = GaussianModel()
        torch.manual_seed(7)
        out, _ = DPMSolver3MSDESampler(model).sample(S=S, batch_size=1, shape=(1, 1, n), eta=1.0, verbose=False,
                                                     timestep_spacing="uniform_trailing")
        assert model.forwards == S
        ref = _solve_3m(ac, S, draws[0].double(), [d.double() for d in draws[1:]])
        d = float((out.double() - ref).abs().max())
        print(f"S={S}: sampler vs independent loop max |diff| {d:.2e}")
        # the sampler's step scalars are fp32 (as DDIM's): at the a = 0 step sqrt(1 - a' - sigma^2) of the rounded values is ~1e-4, not 0
        assert d < 1e-4, S


def test_first_three_steps_are_the_2m_steps(monkeypatch):
    """uniform_trailing: steps 0 and 1 are first order and step 2 is the 2M step, so runs of S <= 4 and the first three steps of
    S = 10 equal the 2M sampler bit for bit (with the fp64 double of both updates)."""
    for S in (1, 2, 3, 4, 10):
        outs = []
        for cls in (DPMSolverSampler, DPMSolver3MSDESampler):
            out, inter, _ = _sample(cls, S, torch.randn(1, 1, 1, 16, generator=torch.Generator().manual_seed(S)), monkeypatch, seed=11)
            outs.append((out, inter["x_inter"]))
        if S <= 4:
            assert torch.equal(outs[0][0], outs[1][0]), S
        else:
            for k in (1, 2, 3):
                assert torch.equal(outs[0][1][k], outs[1][1][k]), k
            assert not torch.equal(outs[0][1][4], outs[1][1][4])


@pytest.mark.parametrize("cls3", [DPMSolver3MSDESampler, DPMSolver3MSDESamplerMultiCond])
def test_sde_std_error_ordering(cls3, monkeypatch):
    """eta = 1: the error of the output's std over 4e5 samples, every solver with the same x_T and noise seeds at each S (Monte Carlo, so
    by ordering, not by value).  The printed line is the table of INTEGRATION.md "Samplers"."""
    ac = _alphas()
    n = 400_000
    std_exact = math.sqrt(ac[0] * S0 * S0 + 1 - ac[0])
    cls2 = DPMSolverSamplerMultiCond if cls3 is DPMSolver3MSDESamplerMultiCond else DPMSolverSampler
    errs = {}
    for S in TABLE_STEPS:
        for k, smp in enumerate((DDIMSampler, cls2, cls3)):
            x_T = torch.randn(1, 1, 1, n, generator=torch.Generator().manual_seed(S))
            out, _, model = _sample(smp, S, x_T, monkeypatch, seed=100 + S)
            assert model.forwards == S
            errs[S, k] = float(out.std()) - std_exact
            if k == 2:
                assert abs(float(out.mean()) - math.sqrt(ac[0]) * MU) < 0.005, S
    for k, name in enumerate(("DDIM eta=1", "DPM-Solver++(2M) SDE", "DPM-Solver++(3M) SDE")):
        print(f"{name}: " + " | ".join(f"S={S} {errs[S, k]:+.3f}" for S in TABLE_STEPS))
    for S in (10, 15, 20):
        assert abs(errs[S, 2]) < abs(errs[S, 1]), S
    assert abs(errs[10, 2]) < abs(errs[50, 0])


def test_generator_is_consumed_like_ddim(monkeypatch):
    _patch(monkeypatch)
    states = []
    for cls in (DDIMSampler, DPMSolver3MSDESampler):
        torch.manual_seed(3)
        cls(GaussianModel()).sample(S=6, batch_size=2, shape=(1, 1, 8), eta=1.0, verbose=False, timestep_spacing="uniform_trailing")
        states.append(torch.get_rng_state())
    assert torch.equal(states[0], states[1])


def test_batch_rows_match_the_single_rows(monkeypatch):
    """B = 2 against each row on its own (_rng_rows): both histories follow the batch."""
    _patch(monkeypatch)
    torch.manual_seed(5)
    b2, _ = DPMSolver3MSDESampler(GaussianModel()).sample(S=8, batch_size=2, shape=(1, 1, 8), eta=1.0, verbose=False,
                                                          timestep_spacing="uniform_trailing")
    for b in range(2):
        torch.manual_seed(5)
        b1, _ = DPMSolver3MSDESampler(GaussianModel()).sample(S=8, batch_size=2, shape=(1, 1, 8), eta=1.0, verbose=False,
                                                              timestep_spacing="uniform_trailing", _rng_rows=(b, b + 1))
        assert torch.equal(b2[b:b + 1], b1), b


@pytest.mark.parametrize("opt", [dict(mask=torch.ones(1)), dict(x0=torch.ones(1)), dict(noise_dropout=0.1), dict(temperature=0.9),
                                 dict(repeat_noise=True), dict(timesteps=5), dict(score_corrector=object()), dict(quantize_x0=True)])
@pytest.mark.parametrize("cls", [DPMSolver3MSDESampler, DPMSolver3MSDESamplerMultiCond])
def test_rejected_options_raise_before_any_forward(opt, cls):
    model = GaussianModel()
    name = next(iter(opt))
    with pytest.raises(NotImplementedError, match=name):
        cls(model).sample(S=5, batch_size=1, shape=(1, 1, 8), eta=1.0, verbose=False, **opt)
    with pytest.raises(NotImplementedError, match="decode"):
        cls(model).decode(torch.zeros(1, 1, 1, 8), None, 2)
    assert model.forwards == 0


@pytest.mark.parametrize("eta", [0.0, 0.5, 0.9999, 2.0])
def test_eta_other_than_one_raises(eta):
    model = GaussianModel()
    for cls in (DPMSolver3MSDESampler, DPMSolver3MSDESamplerMultiCond):
        with pytest.raises(ValueError, match="eta"):
            cls(model).sample(S=5, batch_size=1, shape=(1, 1, 8), eta=eta, verbose=False)
        with pytest.raises(ValueError, match="eta"):          # DDIM's default eta is 0
            cls(model).sample(S=5, batch_size=1, shape=(1, 1, 8), verbose=False)
    assert model.forwards == 0


def test_synthesis_rejects_unknown_sampler_and_eta_before_any_work():
    from viewcrafter_b200 import synthesis

    class NoModel:
        def __getattr__(self, name):
            raise AssertionError(f"touched model.{name}")
    with pytest.raises(ValueError, match="sampler"):
        synthesis.image_guided_synthesis(NoModel(), [""], None, [1, 4, 2, 8, 8], sampler="dpmpp_3m")
    for eta in (0.0, 0.5):
        with pytest.raises(ValueError, match="eta"):
            synthesis.image_guided_synthesis(NoModel(), [""], None, [1, 4, 2, 8, 8], ddim_eta=eta, sampler="dpmpp_3m_sde")
    assert synthesis.SAMPLERS["dpmpp_3m_sde"] == (DPMSolver3MSDESampler, DPMSolver3MSDESamplerMultiCond)
