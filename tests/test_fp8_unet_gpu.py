"""FP8 mode of the full-width U-Net at the baseline sizes 25x40x64 and 25x72x128, with the synthetic weights of
test_zz_baseline_size_gpu.py.

Accuracy gate (self-calibrating, like the 2 * E_ref rule of the fp16 path): the fp32 oracle (oracle/lvdm_oracle.py) is run a second
time with every F.conv2d / F.conv3d / F.linear that the library runs in FP8 fake-quantised -- its input rounded to e4m3 with the
per-tensor just-in-time scale amax / 448, its ORIGINAL weight rounded to e4m3 per output channel -- and the same exclusions (first
conv, last conv, the context K/V projections, and the fp32 embedding MLPs, which are not tap-GEMMs).  With E_fq = |fake-quant - fp32|:

    accept   max|ours_fp8 - fp32| <= 2 * max E_fq   and   mean|ours_fp8 - fp32| <= 2 * mean E_fq

for one forward at t in {999, 499, 19}, for x_prev / pred_x0 of one CFG DDIM step, and for a batch_cfg B=2 forward.  The numbers are
written to $VC_PARITY_OUT/parity_fp8.json when that variable names a directory.  FP8 mode must also be deterministic: eager, graph
replay and a repeated call give the same bits, and switching it off returns to the fp16 results bit for bit.
"""
import json
import os
import re
import types

import pytest
import torch
import torch.nn.functional as F

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
        for p in m.parameters():
            if float(p.detach().abs().max()) == 0.0:
                p.copy_(torch.randn(p.shape, generator=gd, device=dev) * 0.02)
    return m.eval()


def _dump():
    out = os.environ.get("VC_PARITY_OUT")
    if not out:
        return
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "parity_fp8.json"), "w") as f:
            json.dump(_RESULTS, f, indent=1)
    except OSError:
        pass


def _q_act(x):
    amax = float(x.abs().max())
    s = amax / 448.0 if amax > 0 else 1.0
    return (x * (1.0 / s)).clamp(-448, 448).to(torch.float8_e4m3fn).float() * s


def _q_w(w):
    w2 = w.reshape(w.shape[0], -1)
    amax = w2.abs().amax(1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return ((w2 / s[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn).float() * s[:, None]).view(w.shape)


def _fake_quant_F(sd):
    """A stand-in for the oracle's `F` whose conv / linear calls run fake-quantised unless their weight is excluded."""
    excluded = {sd[k].data_ptr() for k in sd if k in ("input_blocks.0.0.weight", "out.2.weight")
                or re.search(r"(time_embed|fps_embedding|emb_layers)\.", k)
                or (re.search(r"attn2\.to_(k|v)(_ip)?\.weight$", k) and sd[k].shape[1] == 1024)}

    def wrap(fn):
        def call(x, w, *a, **k):
            if w.data_ptr() in excluded:
                return fn(x, w, *a, **k)
            return fn(_q_act(x), _q_w(w), *a, **k)
        return call
    ns = types.SimpleNamespace(**{n: getattr(F, n) for n in dir(F) if not n.startswith("_")})
    ns.conv2d, ns.conv3d, ns.linear = wrap(F.conv2d), wrap(F.conv3d), wrap(F.linear)
    return ns


def _oracle_pair(sd, xc, ts, ctx, fs):
    """(fp32 oracle, fake-quant fp32 oracle) outputs of one U-Net forward on the GPU."""
    from oracle import lvdm_oracle as O
    with torch.no_grad(), O.exact_fp32():
        ref32 = O.unet_forward(sd, xc, ts, ctx, fs)
        real_F = O.F
        O.F = _fake_quant_F(sd)
        try:
            reffq = O.unet_forward(sd, xc, ts, ctx, fs)
        finally:
            O.F = real_F
    return ref32, reffq


def _rec(ours, r32, rfq):
    e_fq, err = (rfq - r32).abs(), (ours - r32).abs()
    return dict(max_abs_err=float(err.max()), mean_abs_err=float(err.mean()), e_fq_max=float(e_fq.max()),
                e_fq_mean=float(e_fq.mean()), out_std=float(r32.std()))


@pytest.mark.parametrize("name", list(SIZES))
def test_fp8_accuracy_gate(model, name):
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
    unet.enable_fp8()
    try:
        for t in (999, 499, 19):
            ts = torch.full((1,), t, dtype=torch.long, device="cuda")
            ref32, reffq = _oracle_pair(sd, xc, ts, ctx_c, fs)
            y = unet(xc, ts, context=ctx_c, fs=fs).float()
            res[f"forward_t{t}"] = _rec(y, ref32, reffq)
            print(name, "t=%d" % t, res[f"forward_t{t}"])
            if t == 999:
                keep = (ref32, reffq, ts)
            del ref32, reffq, y
        ref32_c, reffq_c, ts = keep
        ref32_u, reffq_u = _oracle_pair(sd, xc, ts, ctx_u, fs)
        # a batch_cfg B=2 forward (cond + uncond, shared prefix) against the per-branch references
        y2 = unet(torch.cat([xc, xc]), ts.repeat(2), context=torch.cat([ctx_c, ctx_u]), fs=fs.repeat(2), cfg_shared_prefix=True).float()
        res["forward_B2"] = _rec(y2, torch.cat([ref32_c, ref32_u]), torch.cat([reffq_c, reffq_u]))
        print(name, "B=2", res["forward_B2"])
        del y2
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
        pfq, x0_fq = O.ddim_update(x, reffq_c, reffq_u, sc, a, b, noise, 7.5, 0.7)
        for nm, ours, r32, rfq in (("x_prev", x_prev, p32, pfq), ("pred_x0", pred_x0, x0_32, x0_fq)):
            res[f"step999_{nm}"] = _rec(ours, r32, rfq)
            print(name, nm, res[f"step999_{nm}"])
    finally:
        unet.enable_fp8(False)
    _RESULTS[name] = res
    _dump()
    for k, r in res.items():
        assert r["max_abs_err"] <= 2.0 * r["e_fq_max"], (name, k, r)
        assert r["mean_abs_err"] <= 2.0 * r["e_fq_mean"], (name, k, r)


def test_fp8_deterministic_and_switch_back(model):
    unet = model.model.diffusion_model
    H, W = SIZES["ViewCrafter_25_512"][:2]
    g = torch.Generator().manual_seed(3)
    xc = torch.randn(2, 8, T, H, W, generator=g).cuda()
    ctx = torch.randn(2, 333, 1024, generator=g).cuda()
    ts, fs = torch.full((2,), 499, dtype=torch.long, device="cuda"), torch.tensor([10, 10], device="cuda")
    unet.enable_cuda_graph(False)
    y16 = unet(xc, ts, context=ctx, fs=fs)
    unet.enable_fp8()
    eager = [unet(xc, ts, context=ctx, fs=fs) for _ in range(2)]
    unet.enable_cuda_graph(True)
    graphed = [unet(xc, ts, context=ctx, fs=fs) for _ in range(4)]      # eager, capture, replay, replay
    unet.enable_cuda_graph(False)
    assert all(torch.equal(eager[0], y) for y in eager[1:] + graphed)
    assert not torch.equal(eager[0], y16)
    unet.enable_fp8(False)
    assert torch.equal(unet(xc, ts, context=ctx, fs=fs), y16)
