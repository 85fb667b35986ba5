"""Windowed temporal attention (FreeNoise) on the GPU: the kernel, the U-Net, the samplers and several GPUs.

Kernel: `ops.temporal_attn_windowed` against float64 per-window attention blended by the definition, through the blend of the
per-window bounds of `tests/attention_ref.py` (worst |out - ref| / bound <= 1), over windows (16, 25, 32) x strides (1, 4, W), clip
lengths from W + 1 to 346, odd site counts and the level-0 grid; T <= W equal to `ops.temporal_attn`; determinism and independence
from the site count.  U-Net: the model_channels = 64 U-Net against the fp32 oracle with windowed temporal attention
(`tests/window_ref.oracle_window`) within the bounds of `tests/test_unet_gpu.py`.  Samplers: `image_guided_synthesis` with a window on
49- and 160-frame clips against the oracle pipeline fed the same rescheduled x_T; DPM-Solver++(3M) SDE equal to DDIM on first-order
steps.  Several GPUs: `tools/window_check.py` on 2 and 4 ranks (skipped with fewer devices).
"""
import os
import subprocess
import sys

import pytest
import torch

from tests import attention_ref as ar
from tests import window_ref as wr

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_ERR, MEAN_ERR = 0.02, 0.003          # the U-Net forward bounds of test_unet_gpu.py
HW0, HEADS0 = 72 * 128, 5                # level 0 at 576x1024
RUNGS = ["centred", "peaked16", "shift-30", "late-max@last", "v-offset"]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


def _qkv_rows(q, k, v, B, T, sites, heads):
    C = heads * 64
    rows_of = lambda t: t.view(B, sites, T, C).transpose(1, 2).reshape(B * T * sites, C)
    return torch.cat([rows_of(q), rows_of(k), rows_of(v)], 1)


def _run(ops, qkv, B, T, sites, heads, W, S):
    C = heads * 64
    a = torch.empty((B * T * sites, C), device="cuda", dtype=torch.float16)
    for b in range(B):
        rows = slice(b * T * sites, (b + 1) * T * sites)
        ops.temporal_attn_windowed(qkv[rows, :C], qkv[rows, C:2 * C], qkv[rows, 2 * C:], T, sites, heads, W, S, out=a[rows])
    return a


def window_case(ops, rung, B, T, sites, heads, W, S, seed=0):
    """Worst |out - ref| / bound of one windowed launch per batch element, rows at (t * sites + site)."""
    q, k, v = ar.rung_qkv(rung, B * sites, T, T, heads, seed)                    # [B*sites, T, heads, 64]
    a = _run(ops, _qkv_rows(q, k, v, B, T, sites, heads), B, T, sites, heads, W, S)
    assert bool(torch.isfinite(a).all())
    out = a.view(B, T, sites, heads, 64).permute(0, 2, 3, 1, 4).reshape(B * sites, heads, T, 64)
    per = lambda t: t.transpose(1, 2)                                             # [B*sites, heads, T, 64]
    n_win = len(wr.starts(T, W, S))
    step = max(1, (1 << 27) // (heads * n_win * W * 64 * 8 * 4))                  # groups per float64 chunk
    worst = 0.0
    for g0 in range(0, B * sites, step):
        gs = slice(g0, g0 + step)
        ref, bnd = wr.windowed_ref(per(q[gs]), per(k[gs]), per(v[gs]), W, S)
        worst = max(worst, ar.worst_ratio(out[gs], ref, bnd))
    return worst


def _check(r, what):
    print(f"{what}: worst |out - ref| / bound = {r:.3g}")
    assert r <= 1.0, f"{what}: |out - ref| / bound = {r:.4g}"


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("T", ["W+1", 49, 128, 129, 200, 346])
@pytest.mark.parametrize("S", [1, 4, "W"])
@pytest.mark.parametrize("W", [16, 25, 32])
def test_windowed_kernel_vs_f64(ops, W, S, T):
    S = W if S == "W" else S
    T = W + 1 if T == "W+1" else T
    for rung in RUNGS:
        _check(window_case(ops, rung, 1, T, 7, 3, W, S, seed=T + W), f"W={W} S={S} T={T} {rung}")


@pytest.mark.parametrize("sites", [1, 7, 33])
@pytest.mark.parametrize("W,S,T", [(16, 4, 129), (25, 4, 49), (32, 32, 200)])
def test_windowed_kernel_site_counts(ops, W, S, T, sites):
    """3 heads: fewer pairs than warps of one CTA (sites = 1), odd pair counts, and more pairs than warps."""
    for rung in RUNGS:
        _check(window_case(ops, rung, 1, T, sites, 3, W, S, seed=sites), f"W={W} S={S} T={T} sites={sites} {rung}")


@pytest.mark.parametrize("rung", RUNGS)
def test_windowed_kernel_level0(ops, rung):
    """9216 sites x 5 heads, B = 2, at T = 49 with (25, 4): far more pairs than resident warps, so every warp strides."""
    _check(window_case(ops, rung, 2, 49, HW0, HEADS0, 25, 4, seed=43), f"level0 T=49 {rung}")


@pytest.mark.parametrize("W,S", [(16, 4), (25, 1), (32, 32)])
def test_windowed_kernel_is_temporal_attn_up_to_W(ops, W, S):
    for T in sorted({1, 2, 16, W - 1, W}):
        q, k, v = ar.rung_qkv("centred", 33, T, T, 3, seed=T)
        qkv = _qkv_rows(q, k, v, 1, T, 33, 3)
        a = _run(ops, qkv, 1, T, 33, 3, W, S)
        b = ops.temporal_attn(qkv[:, :192], qkv[:, 192:384], qkv[:, 384:], T, 33, 3)
        assert torch.equal(a, b), (W, S, T)


@pytest.mark.parametrize("W,S,T", [(16, 4, 160), (25, 3, 49), (32, 1, 129)])
def test_windowed_kernel_deterministic_and_site_invariant(ops, W, S, T):
    sites, heads = 33, 3
    q, k, v = ar.rung_qkv("centred", sites, T, T, heads, seed=5)
    qkv = _qkv_rows(q, k, v, 1, T, sites, heads)
    a = _run(ops, qkv, 1, T, sites, heads, W, S)
    assert torch.equal(a, _run(ops, qkv, 1, T, sites, heads, W, S))
    for site in (0, 17, 32):                                     # one site alone: its pairs bit-equal to the full launch
        one = _qkv_rows(q[site:site + 1], k[site:site + 1], v[site:site + 1], 1, T, 1, heads)
        alone = _run(ops, one, 1, T, 1, heads, W, S)
        assert torch.equal(alone, a.view(T, sites, -1)[:, site]), site


def test_windowed_kernel_rejects_arguments(ops):
    q = torch.zeros((64, 3 * 64), device="cuda", dtype=torch.float16)
    out = torch.full((64, 64), 7.0, device="cuda", dtype=torch.float16)
    for W, S, msg in [(1, 1, r"W=1 unsupported \(2\.\.32\)"), (33, 4, r"W=33 unsupported \(2\.\.32\)"),
                      (16, 0, r"S=0 unsupported \(1\.\.W=16\)"), (16, 17, r"S=17 unsupported \(1\.\.W=16\)")]:
        with pytest.raises(ops.VcError, match=msg):
            ops.temporal_attn_windowed(q[:, :64], q[:, 64:128], q[:, 128:], 32, 2, 1, W, S, out=out)
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())                              # nothing was launched


# ------------------------------------------------------------------------------------------------ U-Net
def _unet(seed, **over):
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64, **over))
    sd = synth.synth_state_dict(synth.module_shapes(m), seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


def _oracle(sd, window, *args):
    from oracle import lvdm_oracle as O
    torch.set_num_threads(max(1, min(os.cpu_count() or 1, 16)))
    with torch.no_grad(), wr.oracle_window(window):
        return O.unet_forward(sd, *args)


def _err(y, ref, what):
    err = (y.cpu() - ref).abs()
    print(f"{what}: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g}")
    assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR


@pytest.mark.parametrize("T,window", [(49, (25, 4)), (160, (16, 4))])
def test_unet_windowed_shared_prefix_vs_oracle_and_graph_replay(ops, T, window):
    """The shared-CFG-prefix B = 2 forward (context-free prefix incl. init_attn computed once) against the windowed oracle; graph
    replay bit-equal to eager; the window is part of the graph key (switching it off gives the full-attention forward again, where
    full attention exists: T <= 128)."""
    m, sd = _unet(11)
    g = torch.Generator().manual_seed(12)
    x1 = torch.randn(1, 8, T, 8, 8, generator=g)
    ctx = torch.randn(2, 333, 1024, generator=g)
    ref = _oracle(sd, window, torch.cat([x1, x1], 0), torch.tensor([499, 499]), ctx, torch.tensor([10, 10]))
    x, cc = torch.cat([x1, x1], 0).cuda(), ctx.cuda()
    t, fs = torch.full((2,), 499).cuda(), torch.full((2,), 10).cuda()
    m.set_temporal_window(window)
    eager = m(x, t, context=cc, fs=fs, cfg_shared_prefix=True)
    _err(eager, ref, f"T={T} window={window} shared prefix")
    m.enable_cuda_graph()
    for _ in range(3):                                          # eager, capture, replay
        assert torch.equal(m(x, t, context=cc, fs=fs, cfg_shared_prefix=True), eager)
    if T <= 128:
        m.set_temporal_window(None)
        full = m(x, t, context=cc, fs=fs, cfg_shared_prefix=True)
        m.enable_cuda_graph(False)
        assert torch.equal(full, m(x, t, context=cc, fs=fs, cfg_shared_prefix=True))
        assert not torch.equal(full, eager)
    m.enable_cuda_graph(False)


def test_unet_windowed_per_frame_tokens_batch2_vs_oracle(ops):
    """B = 2 at T = 49 with per-frame image tokens (L = 77 + 16 T) and different timesteps."""
    m, sd = _unet(9)
    g = torch.Generator().manual_seed(10)
    T, window = 49, (16, 8)
    x, ctx = torch.randn(2, 8, T, 8, 8, generator=g), torch.randn(2, 77 + 16 * T, 1024, generator=g)
    t, fs = torch.tensor([999, 19]), torch.tensor([10, 10])
    ref = _oracle(sd, window, x, t, ctx, fs)
    y = m.set_temporal_window(window)(x.cuda(), t.cuda(), context=ctx.cuda(), fs=fs.cuda())
    _err(y, ref, "T=49 (16, 8) per-frame tokens B=2")


@pytest.mark.parametrize("fp8", [False, True])
def test_unet_window_not_shorter_than_clip_is_full_attention(ops, fp8):
    """A window of W >= T leaves the forward bit-identical to window off (fp16 and FP8 mode); in FP8 mode a real window runs."""
    m, _ = _unet(13)
    g = torch.Generator().manual_seed(14)
    T = 25
    x, ctx = torch.randn(3, 8, T, 8, 8, generator=g).cuda(), torch.randn(3, 333, 1024, generator=g).cuda()
    t, fs = torch.tensor([999, 500, 19]).cuda(), torch.full((3,), 10).cuda()
    m.enable_fp8(fp8)
    off = m(x, t, context=ctx, fs=fs)
    for window in ((25, 4), (32, 32)):
        assert torch.equal(m.set_temporal_window(window)(x, t, context=ctx, fs=fs), off), window
    on = m.set_temporal_window((16, 4))(x, t, context=ctx, fs=fs)
    assert bool(torch.isfinite(on).all()) and not torch.equal(on, off)
    m.set_temporal_window(None).enable_fp8(False)


# ------------------------------------------------------------------------------------------------ samplers
def _pipeline_model():
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=dict(VAE_DDCONFIG, ch=32), embed_dim=4), base_scale=0.7).eval()
    sd = synth.synth_state_dict(synth.module_shapes(model.model.diffusion_model), seed=71)
    model.model.diffusion_model.load_state_dict(sd, strict=True)
    sdv = synth.synth_state_dict(synth.module_shapes(model.first_stage_model), seed=72)
    model.first_stage_model.load_state_dict(sdv, strict=True)
    model = model.cuda()
    g = torch.Generator().manual_seed(73)
    W_img, txt, txt_empty = torch.randn(3 * 4 * 4, 256 * 8, generator=g) * 0.1, torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)
    W_d, txt_d, txt_empty_d = W_img.cuda(), txt.cuda(), txt_empty.cuda()
    model.embedder = lambda img: torch.nn.functional.adaptive_avg_pool2d(img, 4).reshape(img.shape[0], 1, -1)
    model.image_proj_model = lambda e: (e @ (W_d if e.is_cuda else W_img)).reshape(e.shape[0], 256, 8).repeat(1, 1, 128)
    model.get_learned_conditioning = lambda prompts: torch.cat([txt_empty_d if p == "" else txt_d for p in prompts], 0)
    model.uncond_type = "empty_seq"
    return model, sd, sdv, txt, txt_empty


@pytest.mark.parametrize("T,window,steps", [(49, (25, 4), 3), (160, (16, 4), 2)])
def test_image_guided_synthesis_windowed_vs_oracle(T, window, steps):
    """image_guided_synthesis(temporal_window=...) (VAE encode, batched CFG DDIM with graph replay, VAE decode) against the oracle
    pipeline with windowed temporal attention, fed the same draws with x_T rescheduled by the independent restatement.  The U-Net's
    window is restored afterwards, and the CPU generator ends where the encode's own draws leave it (the rescheduling uses none)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import lvdm_oracle as O
    from viewcrafter_b200.synthesis import image_guided_synthesis
    model, sd, sdv, txt, txt_empty = _pipeline_model()
    unet = model.model.diffusion_model
    g = torch.Generator().manual_seed(75)
    H, Wd = 8, 8
    videos = torch.rand(1, 3, T, 8 * H, 8 * Wd, generator=g) * 2 - 1
    shape = (1, 4, T, H, Wd)
    torch.manual_seed(74)
    out = image_guided_synthesis(model, ["a photo"], videos.cuda(), list(shape), n_samples=1, ddim_steps=steps, ddim_eta=1.0,
                                 unconditional_guidance_scale=7.5, fs=10, text_input=True, timestep_spacing="uniform_trailing",
                                 guidance_rescale=0.7, condition_index=[0], temporal_window=window, window_seed=3)
    cpu_state = torch.get_rng_state()
    assert unet.temporal_window is None
    assert out.shape == (1, 1, 3, T, 8 * H, 8 * Wd) and bool(torch.isfinite(out).all())
    torch.manual_seed(74)
    enc_noise = [torch.randn(1, 4, H, Wd) for _ in range(T)]
    assert torch.equal(torch.get_rng_state(), cpu_state)
    img = videos[:, :, 0]
    ctx = lambda t, im: torch.cat([t, model.image_proj_model(model.embedder(im))], 1)
    ctx_c, ctx_u = ctx(txt, img), ctx(txt_empty, torch.zeros_like(img))
    fs = torch.tensor([10])
    torch.set_num_threads(max(1, min(os.cpu_count() or 1, 16)))
    with torch.no_grad():
        cc = O.encode_first_stage(sdv, videos, enc_noise)
    sched = O.model_schedule(base_scale=0.7)

    def model_fn(x, t, cond):
        with torch.no_grad(), wr.oracle_window(window):
            return O.unet_forward(sd, torch.cat([x, cc], 1), t, cond, fs)

    x_T = wr.reschedule(torch.randn(shape, device="cuda").cpu(), *window, seed=3)
    noises = [torch.randn(shape, device="cuda").cpu() for _ in range(steps)]
    ref, _ = O.ddim_sample(model_fn, sched, shape, steps, ctx_c, ctx_u, x_T, noises)
    with torch.no_grad():
        ref_img = O.decode_first_stage(sdv, ref)
    err = (out[:, 0].cpu() - ref_img).abs()
    print(f"synthesis T={T} window={window}: mean err {float(err.mean()):.4g} max {float(err.max()):.4g} ref std {float(ref_img.std()):.3g}")
    assert float(err.mean()) < 0.05 * max(1.0, float(ref_img.std()))


@pytest.mark.parametrize("three_way", [False, True])
def test_dpmpp_3m_sde_windowed_first_order_steps_equal_ddim(three_way):
    """Both steps of a 2-step DPM-Solver++(3M) SDE run are first order: with a window (and the rescheduled x_T it draws) the run is
    bit-identical to DDIM with the same seed."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from tests.test_dpm_solver_gpu import _ld_model
    from viewcrafter_b200 import ddim, ddim_multiplecond, dpm_solver
    model = _ld_model()
    model.model.diffusion_model.set_temporal_window((16, 4))
    g = torch.Generator().manual_seed(42)
    shape = (1, 4, 49, 8, 8)
    cc = torch.randn(shape, generator=g).cuda()
    c, uc, ui = ({"c_crossattn": [torch.randn(1, 333, 1024, generator=g).cuda()], "c_concat": [cc]} for _ in range(3))
    classes = (ddim_multiplecond.DDIMSampler, dpm_solver.DPMSolver3MSDESamplerMultiCond) if three_way else \
        (ddim.DDIMSampler, dpm_solver.DPMSolver3MSDESampler)
    outs = []
    for cls in classes:
        kw = dict(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui) if three_way else {}
        torch.manual_seed(43)
        out, inter = cls(model, batch_cfg=True).sample(
            S=2, batch_size=1, shape=shape[1:], conditioning=c, eta=1.0, verbose=False, log_every_t=1, window_seed=5,
            unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=torch.tensor([10]).cuda(),
            timestep_spacing="uniform_trailing", guidance_rescale=0.7, **kw)
        outs.append((out, inter["x_inter"][0], inter["pred_x0"][-1]))
    (a, xa, pa), (b, xb, pb) = outs
    torch.manual_seed(43)
    drawn = torch.randn(shape, device="cuda")
    assert torch.equal(xa, wr.reschedule(drawn.cpu(), 16, 4, seed=5).cuda()) and torch.equal(xa, xb)
    assert a.shape == shape and bool(torch.isfinite(a).all())
    assert torch.equal(a, b) and torch.equal(pa, pb)


# ------------------------------------------------------------------------------------------------ several GPUs
@pytest.mark.parametrize("world", [2, 4])
def test_windowed_multi_gpu(world):
    """tools/window_check.py: the frame-sharded windowed forward at T = 160 against one GPU, reproducible-mode bit-identity on
    1 / 2 / 4 GPUs, and replica groups R = 2 equal to the one-GPU image_guided_synthesis call."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} CUDA devices")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29547", os.path.join(ROOT, "tools", "window_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1700)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0 and "WINDOW_CHECK_OK" in r.stdout
