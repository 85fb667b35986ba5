"""DPM-Solver++(2M) sampler (viewcrafter_b200.dpm_solver) on the CPU:
  * the host coefficients (schedule.dpm_coefficients) against an independent fp64 restatement in log-SNR form, for every spacing;
  * the sampler loop on an analytic problem -- data x0 ~ N(0.5, 0.8^2) on ViewCrafter's schedule (zero terminal SNR,
    uniform_trailing, v-prediction), whose optimal denoiser and exact probability-flow ODE solution are closed form -- with
    ops.dpm_update / ops.ddim_update replaced by the fp64 restatement below (dpm_update_f64, also the GPU test's reference);
  * the options the sampler rejects, before any forward."""
import math

import numpy as np
import pytest
import torch

from viewcrafter_b200 import ops, schedule
from viewcrafter_b200.ddim import DDIMSampler
from viewcrafter_b200.dpm_solver import DPMSolverSampler, DPMSolverSamplerMultiCond

MU, S0 = 0.5, 0.8
SPACINGS = ("uniform", "uniform_trailing", "quad")
# max |x_out - x_exact| over 101 values of x_T in [-3, 3], as printed in INTEGRATION.md: S -> (DDIM eta=0, DPM-Solver++(2M))
ODE_TABLE = {10: ("0.361", "0.184"), 20: ("0.193", "0.062"), 25: ("0.157", "0.044"), 50: ("0.082", "0.016"), 100: ("0.042", "0.0051")}


def dpm_update_f64(x, v_cond, v_uncond, noise, sc, x0_hist, v_uncond_img=None, cfg_img=0.0):
    """fp64 restatement of ops.dpm_update (one call = one sample: the guidance-rescale stds run over the whole tensor).  Writes this
    step's x0 (before the dynamic rescale) into x0_hist and returns fp64 (x_prev, pred_x0)."""
    d = lambda t: None if t is None else t.double()
    x, c, u, vi, nz = d(x), d(v_cond), d(v_uncond), d(v_uncond_img), d(noise)
    m = c
    if u is not None and sc["cfg_scale"] != 1.0:
        s = sc["cfg_scale"]
        m = u + s * (c - u) if vi is None else u + cfg_img * (vi - u) + s * (c - vi)
        g = sc["guidance_rescale"]
        if g > 0:
            m = g * (m * (c.std() / m.std())) + (1 - g) * m
    x0 = sc["sqrt_ac_t"] * x - sc["sqrt_1mac_t"] * m
    e_t = sc["sqrt_ac_t"] * m + sc["sqrt_1mac_t"] * x
    p0 = x0 * (sc["prev_scale_t"] / sc["scale_t"])
    a_prev, sig = sc["a_prev"], sc["sigma_t"]
    x_prev = math.sqrt(a_prev) * p0 + math.sqrt(max(1.0 - a_prev - sig * sig, 0.0)) * e_t + sig * nz
    if sc["c_hist"] != 0.0:
        x_prev = x_prev + sc["c_hist"] * (x0 - x0_hist.double())
    x0_hist.copy_(x0)
    return x_prev, p0


def ddim_update_f64(x, v_cond, v_uncond, noise, sc, v_uncond_img=None, cfg_img=0.0):
    return dpm_update_f64(x, v_cond, v_uncond, noise, dict(sc, c_hist=0.0), torch.empty(x.shape, dtype=torch.float64),
                          v_uncond_img, cfg_img)


def lam(a):
    """log-SNR / 2 in the alpha / sigma form: log(alpha / sigma); -inf at a = 0."""
    return -math.inf if a == 0 else math.log(math.sqrt(a) / math.sqrt(1.0 - a))


def coefficients_ref(ac, ts, eta):
    """c of every step in sampling order (first step first), restated from the definitions with alpha and sigma."""
    ts = [int(t) for t in ts[::-1]]
    targets = ts[1:] + [None]
    out = []
    for i, t in enumerate(ts):
        a, a_next = ac[t], (ac[targets[i]] if targets[i] is not None else ac[0])
        if i == 0 or i == len(ts) - 1 or ac[ts[i - 1]] == 0.0:
            out.append(0.0)
            continue
        h, h_prev = lam(a_next) - lam(a), lam(a) - lam(ac[ts[i - 1]])
        if h == 0.0 or h_prev == 0.0:
            out.append(0.0)
            continue
        ratio = (math.sqrt(1 - a_next) / math.sqrt(1 - a)) * (math.sqrt(a) / math.sqrt(a_next))     # exp(-h)
        out.append(math.sqrt(a_next) * (1.0 - ratio ** (1 + eta)) / (2.0 * h_prev / h))
    return np.asarray(out[::-1])                   # DDIM index order


def _alphas():
    return schedule.model_buffers()["alphas_cumprod"].double().numpy()


@pytest.mark.parametrize("spacing", SPACINGS)
@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_coefficients_match_the_log_snr_restatement(spacing, eta):
    ac = _alphas()
    for S in (1, 2, 3, 10, 25, 50):
        ts = schedule.ddim_timesteps(spacing, S, 1000)
        if ts.max() >= 1000:                 # "uniform" at S = 3 reaches t = 1000: DDIM's own tables fail there (the reference's too)
            for f in (lambda: schedule.ddim_parameters(torch.from_numpy(ac), ts, eta), lambda: schedule.dpm_coefficients(ac, ts, eta)):
                with pytest.raises(IndexError):
                    f()
            continue
        S = len(ts)
        c = schedule.dpm_coefficients(ac, ts, eta)
        ref = coefficients_ref(ac, ts, eta)
        assert c.shape == (S,) and c.dtype == np.float64 and np.all(np.isfinite(c)), (spacing, S)
        assert np.array_equal(c == 0, ref == 0), (spacing, S, c, ref)
        np.testing.assert_allclose(c, ref, rtol=1e-12, atol=0, err_msg=f"{spacing} S={S}")
        assert c[0] == 0.0 and c[-1] == 0.0                     # the last and the first step are first order
        if S >= 3:
            first_order = {0, S - 1} | ({S - 2} if ac[ts[-1]] == 0 else set())
            assert {j for j in range(S) if c[j] == 0} == first_order or spacing == "quad", (spacing, S, c)


def test_zero_terminal_snr_makes_the_first_two_trailing_steps_first_order():
    ac = _alphas()
    assert ac[999] == 0.0
    for eta in (0.0, 1.0):
        c = schedule.dpm_coefficients(ac, schedule.ddim_timesteps("uniform_trailing", 10, 1000), eta)
        assert c[9] == 0 and c[8] == 0 and c[0] == 0 and np.all(c[1:8] > 0)


class GaussianModel:
    """The v-prediction of the optimal denoiser for data x0 ~ N(MU, S0^2) on ViewCrafter's schedule (zero terminal SNR, no dynamic
    rescale): the stub model object the samplers run on."""
    parameterization = "v"
    use_dynamic_rescale = False

    def __init__(self):
        for k, v in schedule.model_buffers(dynamic_rescale=False).items():
            setattr(self, k, v)
        self.num_timesteps = 1000
        self.forwards = 0

    def apply_model(self, x, t, c, **kwargs):
        self.forwards += 1
        step = int(t[0])
        a = float(self.alphas_cumprod[step])
        al, sg = float(self.sqrt_alphas_cumprod[step]), float(self.sqrt_one_minus_alphas_cumprod[step])
        xd = x.double()
        x0 = MU + math.sqrt(a) * S0 * S0 / (a * S0 * S0 + 1 - a) * (xd - math.sqrt(a) * MU)
        return (al * xd - x0) / sg                 # so that sqrt_ac x - sqrt_1mac v = x0


def _solve_ref(ac, S, second_order, x, eta=0.0, noises=None):
    """Independent fp64 restatement of DDIM (eta 0 / 1) and DPM-Solver++(2M) on the Gaussian problem, last step first order.  The
    latent and the x0 history are held in fp32 between steps, as the sampler holds them."""
    ts = [int(t) for t in schedule.ddim_timesteps("uniform_trailing", S, 1000)[::-1]]
    prev = h_prev = None
    for i, t in enumerate(ts):
        x = x.float().double()
        a, a_next = ac[t], (ac[ts[i + 1]] if i + 1 < S else ac[0])
        x0 = MU + math.sqrt(a) * S0 * S0 / (a * S0 * S0 + 1 - a) * (x - math.sqrt(a) * MU)
        eps = (x - math.sqrt(a) * x0) / math.sqrt(1 - a)
        sig = eta * math.sqrt((1 - a_next) / (1 - a) * (1 - a / a_next))
        xn = math.sqrt(a_next) * x0 + math.sqrt(max(1 - a_next - sig * sig, 0.0)) * eps
        if noises is not None:
            xn = xn + sig * noises[i]
        h = lam(a_next) - lam(a)
        if second_order and prev is not None and math.isfinite(h_prev) and i < S - 1:
            xn = xn + math.sqrt(a_next) * -math.expm1(-(1 + eta) * h) / (2 * h_prev / h) * (x0 - prev)
        prev, h_prev, x = x0.float().double(), h, xn
    return x


def _sample(cls, S, x_T, eta, monkeypatch, seed=0):
    monkeypatch.setattr(ops, "dpm_update", dpm_update_f64)
    monkeypatch.setattr(ops, "ddim_update", ddim_update_f64)
    model = GaussianModel()
    torch.manual_seed(seed)
    kw = dict(unconditional_conditioning_img_nonetext=None) if cls is DPMSolverSamplerMultiCond else {}
    out, inter = cls(model).sample(S=S, batch_size=1, shape=tuple(x_T.shape[1:]), x_T=x_T, eta=eta, verbose=False,
                                   timestep_spacing="uniform_trailing", **kw)
    return out.double(), inter, model


def _exact(ac, x_T):
    return math.sqrt(ac[0]) * MU + math.sqrt(ac[0] * S0 * S0 + 1 - ac[0]) * x_T


def test_ode_convergence_on_the_gaussian_problem(monkeypatch):
    ac = _alphas()
    x_T = torch.linspace(-3, 3, 101, dtype=torch.float64).reshape(1, 1, 1, 101)
    exact = _exact(ac, x_T)
    errs = {}
    for S, (tab_ddim, tab_dpm) in ODE_TABLE.items():
        for k, (cls, order2, tab) in enumerate(((DDIMSampler, False, tab_ddim), (DPMSolverSampler, True, tab_dpm))):
            out, inter, model = _sample(cls, S, x_T.float(), 0.0, monkeypatch)
            ref = _solve_ref(ac, S, order2, x_T.float().double())
            assert model.forwards == S
            d = float((out - ref).abs().max())
            err = float((out - exact).abs().max())
            print(f"S={S} {cls.__name__}: max error {err:.6f} (table {tab}), sampler vs fp64 restatement {d:.2e}")
            # 1e-6 relative to the output (|x| reaches 3): the sampler's step scalars are DDIM's fp32 values, the restatement's fp64
            assert d < 1e-6 * float(ref.abs().max()), (S, cls.__name__, d)
            assert abs(err - float(tab)) <= 0.5 * 10.0 ** -len(tab.split(".")[1]), (S, cls.__name__, err, tab)   # rounds to the table
            errs[S, k] = err
    for S in ODE_TABLE:
        assert errs[S, 1] < errs[S, 0]
    assert errs[20, 1] < errs[50, 0]


@pytest.mark.parametrize("cls", [DPMSolverSampler, DPMSolverSamplerMultiCond])
def test_sde_std_error_ordering(cls, monkeypatch):
    """eta = 1: the error of the output's std over 4e5 samples (Monte Carlo, so by ordering, not by value)."""
    ac = _alphas()
    n = 400_000
    std_exact = math.sqrt(ac[0] * S0 * S0 + 1 - ac[0])
    errs = {}
    for S in (10, 20, 25, 50):
        for k, smp in enumerate((DDIMSampler, cls)):
            x_T = torch.randn(1, 1, 1, n, generator=torch.Generator().manual_seed(S))
            out, _, _ = _sample(smp, S, x_T, 1.0, monkeypatch, seed=100 + S)
            errs[S, k] = float(out.std()) - std_exact
        print(f"S={S}: std error DDIM eta=1 {errs[S, 0]:+.4f}, DPM-Solver++(2M) SDE {errs[S, 1]:+.4f}")
        assert abs(errs[S, 1]) < abs(errs[S, 0]), S
    assert abs(errs[20, 1]) < abs(errs[50, 0])


def test_sde_sampler_matches_the_restatement_with_its_own_noise(monkeypatch):
    """eta = 1 with the draws the sampler makes (x_T, then one noise tensor per step, like DDIMSampler.sample)."""
    ac = _alphas()
    S, n = 10, 64
    torch.manual_seed(7)
    draws = [torch.randn(1, 1, 1, n) for _ in range(S + 1)]
    monkeypatch.setattr(ops, "dpm_update", dpm_update_f64)
    torch.manual_seed(7)
    out, _ = DPMSolverSampler(GaussianModel()).sample(S=S, batch_size=1, shape=(1, 1, n), eta=1.0, verbose=False,
                                                      timestep_spacing="uniform_trailing")
    ref = _solve_ref(ac, S, True, draws[0].double(), eta=1.0, noises=[d.double() for d in draws[1:]])
    # the sampler's step scalars are fp32 (as DDIM's): at the a = 0 step sqrt(1 - a' - sigma^2) of the rounded values is ~1e-4, not 0
    assert float((out.double() - ref).abs().max()) < 1e-4


def test_generator_is_consumed_like_ddim(monkeypatch):
    monkeypatch.setattr(ops, "dpm_update", dpm_update_f64)
    monkeypatch.setattr(ops, "ddim_update", ddim_update_f64)
    states = []
    for cls in (DDIMSampler, DPMSolverSampler):
        for eta in (0.0, 1.0):
            torch.manual_seed(3)
            cls(GaussianModel()).sample(S=5, batch_size=2, shape=(1, 1, 8), eta=eta, verbose=False, timestep_spacing="uniform_trailing")
            states.append(torch.get_rng_state())
    assert all(torch.equal(s, states[0]) for s in states)


def test_first_order_runs_equal_ddim(monkeypatch):
    """S = 1 and 2 under uniform_trailing (every step first order), and the first two steps of S = 10, with the fp64 double."""
    monkeypatch.setattr(ops, "dpm_update", dpm_update_f64)
    monkeypatch.setattr(ops, "ddim_update", ddim_update_f64)
    for S in (1, 2, 10):
        for eta in (0.0, 1.0):
            outs = []
            for cls in (DDIMSampler, DPMSolverSampler):
                torch.manual_seed(11)
                out, inter = cls(GaussianModel()).sample(S=S, batch_size=1, shape=(1, 1, 16), eta=eta, verbose=False, log_every_t=1,
                                                         timestep_spacing="uniform_trailing")
                outs.append((out, inter["x_inter"]))
            if S < 10:
                assert torch.equal(outs[0][0], outs[1][0])
            else:
                for k in (1, 2):
                    assert torch.equal(outs[0][1][k], outs[1][1][k])
                assert not torch.equal(outs[0][0], outs[1][0])


@pytest.mark.parametrize("opt", [dict(mask=torch.ones(1)), dict(x0=torch.ones(1)), dict(noise_dropout=0.1), dict(temperature=0.9),
                                 dict(repeat_noise=True), dict(timesteps=5), dict(score_corrector=object()), dict(quantize_x0=True)])
def test_rejected_options_raise_before_any_forward(opt):
    model = GaussianModel()
    name = next(iter(opt))
    with pytest.raises(NotImplementedError, match=name):
        DPMSolverSampler(model).sample(S=5, batch_size=1, shape=(1, 1, 8), verbose=False, **opt)
    assert model.forwards == 0


@pytest.mark.parametrize("eta", [0.5, 0.0001, 2.0])
def test_eta_other_than_zero_or_one_raises(eta):
    model = GaussianModel()
    for cls in (DPMSolverSampler, DPMSolverSamplerMultiCond):
        with pytest.raises(ValueError, match="eta"):
            cls(model).sample(S=5, batch_size=1, shape=(1, 1, 8), eta=eta, verbose=False)
    assert model.forwards == 0


def test_synthesis_rejects_unknown_sampler_and_eta_before_any_work():
    from viewcrafter_b200 import synthesis

    class NoModel:
        def __getattr__(self, name):
            raise AssertionError(f"touched model.{name}")
    with pytest.raises(ValueError, match="sampler"):
        synthesis.image_guided_synthesis(NoModel(), [""], None, [1, 4, 2, 8, 8], sampler="euler")
    with pytest.raises(ValueError, match="eta"):
        synthesis.image_guided_synthesis(NoModel(), [""], None, [1, 4, 2, 8, 8], ddim_eta=0.5, sampler="dpmpp_2m")
    assert synthesis.SAMPLERS["dpmpp_2m"] == (DPMSolverSampler, DPMSolverSamplerMultiCond)
