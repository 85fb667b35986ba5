"""Parity AT THE BASELINE.json SIZES (SURVEY.md 8d, configs 1-3): the full-width U-Net (model_channels 320) on
latents 25x4x40x64 (ViewCrafter_25_512) and 25x4x72x128 (ViewCrafter_25, the headline), CUDA path vs the oracle.

The fp32 CPU oracle needs minutes per forward at these sizes, so the SAME oracle code runs on the GPU here: fp32 with
TF32 disabled (``O.exact_fp32``), the reference's naive attention evaluated in batch chunks (``oracle/lvdm_oracle.py``).
Tolerance is the self-calibrating rule of SURVEY.md 8(d) -- the reference states none:

    E_ref = | oracle under torch.autocast(fp16)  -  oracle in fp32 |     (what the reference's own fp16 mode costs,
                                                                           viewcrafter.py:98)
    accept   max|ours - fp32| <= 2 * max E_ref   and   mean|ours - fp32| <= 2 * mean E_ref

checked for one forward at t in {999, 499, 19} and for x_{t-1} / pred_x0 of one full CFG DDIM step (cfg 7.5, guidance
rescale 0.7, eta 1, the 50-step uniform_trailing schedule) with the same noise tensor on both sides.  DDIM indexing is
checked bit-exactly elsewhere (tests/test_schedule_cpu.py, tests/test_oracle_golden.py).  The measured numbers are
written to $VC_PARITY_OUT/parity_baseline_sizes.json when that variable names a directory.
"""
import json
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]

T = 25
SIZES = {"ViewCrafter_25_512": (40, 64, 0.7), "ViewCrafter_25": (72, 128, 0.3)}
_RESULTS = {}


@pytest.fixture(scope="module")
def model():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.diffusion import LatentDiffusion
    dev = torch.device("cuda")
    torch.manual_seed(0)
    with torch.device(dev):
        m = LatentDiffusion(UNET_PARAMS, None, base_scale=0.3)
    gd = torch.Generator(device=dev).manual_seed(1)
    with torch.no_grad():
        for p in m.parameters():                                       # zero-initialised layers would make the output exactly 0
            if float(p.detach().abs().max()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=gd, device=dev) * 0.02)
    return m.eval()


def _dump():
    out = os.environ.get("VC_PARITY_OUT")
    if not out:
        return
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "parity_baseline_sizes.json"), "w") as f:
            json.dump(_RESULTS, f, indent=1)
    except OSError:
        pass


def _oracle_pair(sd, xc, ts, ctx, fs):
    """(fp32 oracle, fp16-autocast oracle) outputs of one U-Net forward on the GPU."""
    from oracle import lvdm_oracle as O
    with torch.no_grad(), O.exact_fp32():
        ref32 = O.unet_forward(sd, xc, ts, ctx, fs)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        ref16 = O.unet_forward(sd, xc, ts, ctx, fs).float()
    return ref32, ref16


@pytest.mark.parametrize("name", list(SIZES))
def test_unet_forward_and_ddim_step_at_baseline_size(model, name):
    from oracle import lvdm_oracle as O
    from viewcrafter_b200.ddim import DDIMSampler
    H, W, base_scale = SIZES[name]
    unet = model.model.diffusion_model
    sd = {k: v.detach() for k, v in unet.state_dict().items()}
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 4, T, H, W, generator=g).cuda()
    cc = torch.randn(1, 4, T, H, W, generator=g).cuda()
    ctx_c, ctx_u = torch.randn(1, 333, 1024, generator=g).cuda(), torch.randn(1, 333, 1024, generator=g).cuda()
    fs = torch.tensor([10], device="cuda")
    xc = torch.cat([x, cc], 1)
    res = {}
    for t in (999, 499, 19):
        ts = torch.full((1,), t, dtype=torch.long, device="cuda")
        ref32, ref16 = _oracle_pair(sd, xc, ts, ctx_c, fs)
        y = unet(xc, ts, context=ctx_c, fs=fs).float()
        e_ref, err = (ref16 - ref32).abs(), (y - ref32).abs()
        r = dict(max_abs_err=float(err.max()), mean_abs_err=float(err.mean()), e_ref_max=float(e_ref.max()),
                 e_ref_mean=float(e_ref.mean()), out_std=float(ref32.std()))
        res[f"forward_t{t}"] = r
        print(name, "t=%d" % t, r)
        if t == 999:
            keep = (ref32, ref16, ts)
        del ref32, ref16, y
    # one CFG DDIM step from t=999 (index 49): x_prev / pred_x0 with the same noise draw on both sides
    ref32_c, ref16_c, ts = keep
    ref32_u, ref16_u = _oracle_pair(sd, xc, ts, ctx_u, fs)
    sched = {k: v.cuda() for k, v in O.model_schedule(base_scale=base_scale).items()}
    tab = O.ddim_tables(sched, 50, "uniform_trailing", 1.0)
    model.scale_arr = sched["scale_arr"]
    smp = DDIMSampler(model, batch_cfg=True)
    smp.make_schedule(50, "uniform_trailing", 1.0, verbose=False)
    c = {"c_crossattn": [ctx_c], "c_concat": [cc]}
    uc = {"c_crossattn": [ctx_u], "c_concat": [cc]}
    torch.manual_seed(5)
    x_prev, pred_x0 = smp.p_sample_ddim(x, c, ts, index=49, unconditional_guidance_scale=7.5, unconditional_conditioning=uc,
                                        fs=fs, guidance_rescale=0.7, _step=999)
    torch.manual_seed(5)
    noise = torch.randn(x.shape, device="cuda")
    sc = O.step_scalars(tab, 49)
    a, b = sched["sqrt_alphas_cumprod"][999].item(), sched["sqrt_one_minus_alphas_cumprod"][999].item()
    p32, x0_32 = O.ddim_update(x, ref32_c, ref32_u, sc, a, b, noise, 7.5, 0.7)
    p16, x0_16 = O.ddim_update(x, ref16_c, ref16_u, sc, a, b, noise, 7.5, 0.7)
    for nm, ours, r32, r16 in (("x_prev", x_prev, p32, p16), ("pred_x0", pred_x0, x0_32, x0_16)):
        e_ref, err = (r16 - r32).abs(), (ours - r32).abs()
        res[f"step999_{nm}"] = dict(max_abs_err=float(err.max()), mean_abs_err=float(err.mean()), e_ref_max=float(e_ref.max()),
                                    e_ref_mean=float(e_ref.mean()), out_std=float(r32.std()))
        print(name, nm, res[f"step999_{nm}"])
    _RESULTS[name] = res
    _dump()
    for k, r in res.items():
        assert r["max_abs_err"] <= 2.0 * r["e_ref_max"], (name, k, r)
        assert r["mean_abs_err"] <= 2.0 * r["e_ref_mean"], (name, k, r)
