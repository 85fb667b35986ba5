"""FIFO-Diffusion diagonal denoising on the GPU: the per-frame DDIM update kernel, the U-Net with per-frame timesteps, the diagonal
schedule pinned to DDIM on a frame-local model, and image_guided_synthesis(fifo=f) against the oracle pipeline.

Kernel: ops.ddim_update_frames against the float64 restatement of tests/fifo_ref.py within 16 fp32 ulps of the summed magnitudes plus
the square-root term of tests/test_sampler_sweep_gpu.py, over T in {1, 16, 25, 128} with distinct per-frame scalars from a real schedule
(the last frame at a = 0); with every frame's scalars equal, ops.ddim_update bit for bit.  U-Net: the model_channels = 64 model of
tests/test_unet_gpu.py; [B, T] timesteps that are all equal give the [B] forward bit for bit; distinct ones match
fifo_ref.unet_forward_frames within that file's bounds."""
import os

import pytest
import torch

from tests import fifo_ref as fr
from tests.test_sampler_sweep_gpu import _dir_error

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
EPS32 = 2.0 ** -23
MAX_ERR, MEAN_ERR = 0.02, 0.003          # the U-Net forward bounds of test_unet_gpu.py
CFG, CFG_IMG = 7.5, 2.0


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


class _Sched:
    """The schedule attributes DDIMSampler.make_schedule reads."""
    parameterization = "v"

    def __init__(self, dynamic=True):
        from viewcrafter_b200 import schedule
        self.use_dynamic_rescale = dynamic
        for k, v in schedule.model_buffers(base_scale=0.7, dynamic_rescale=dynamic).items():
            setattr(self, k, v)
        self.num_timesteps = 1000


def _frames(T, eta, dynamic, three_way=False):
    """Distinct per-frame step scalars of a real uniform_trailing schedule: the last T indices of S = max(T, 4) steps, so the last frame
    is the a = 0 step."""
    from viewcrafter_b200 import ddim, ddim_multiplecond
    smp = (ddim_multiplecond.DDIMSampler if three_way else ddim.DDIMSampler)(_Sched(dynamic))
    S = max(T, 4)
    smp.make_schedule(S, "uniform_trailing", eta, verbose=False)
    return [smp.step_scalars(k, int(smp.ddim_timesteps[k])) for k in range(S - T, S)]


def _inputs(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(shape, generator=g) * s for s in (1.0, 1.0, 1.2, 1.1, 1.0)]         # x, v_cond, v_uncond, v_uncond_img, noise


@pytest.mark.parametrize("T", [1, 16, 25, 128])
@pytest.mark.parametrize("three_way", [False, True])
@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_update_frames_vs_f64(T, three_way, eta):
    from viewcrafter_b200 import ops
    shape = (2, 4, T, 5, 7)
    x, vc, vu, vi, nz = _inputs(shape, T)
    m_mag = (vu.abs() + CFG_IMG * (vi.abs() + vu.abs()) + CFG * (vc.abs() + vi.abs()) if three_way
             else vu.abs() + CFG * (vc.abs() + vu.abs())).double()
    worst = 0.0
    for dynamic in (False, True):
        frames = _frames(T, eta, dynamic, three_way)
        assert frames[-1]["sqrt_ac_t"] == 0.0
        for rescale in (0.0, 0.7):
            sc = dict(cfg_scale=CFG, guidance_rescale=rescale)
            kw = dict(v_uncond_img=vi, cfg_img=CFG_IMG) if three_way else {}
            xp, p0 = ops.ddim_update_frames(x.cuda(), vc.cuda(), vu.cuda(), nz.cuda(), sc, frames,
                                            **{k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
            rx, rp = fr.ddim_update_frames_f64(x, vc, vu, nz, sc, frames, **kw)
            col = lambda vals: torch.tensor(vals, dtype=torch.float64).view(1, 1, -1, 1, 1)
            resc = col([max(1.0, fm["prev_scale_t"] / fm["scale_t"]) for fm in frames])
            tol = 16 * EPS32 * (x.double().abs() + m_mag + nz.double().abs()) * resc
            tol_x = tol + col([_dir_error(fm) for fm in frames]) * (x.double().abs() + m_mag)
            for name, got, ref, bound in (("x_prev", xp, rx, tol_x), ("pred_x0", p0, rp, tol)):
                g = got.cpu().double()
                assert bool(torch.isfinite(g).all()), name
                ratio = float(((g - ref).abs() / bound).max())
                worst = max(worst, ratio)
                assert ratio <= 1.0, f"{name}: error / bound {ratio:.3g} (T={T}, dynamic={dynamic}, rescale={rescale})"
    print(f"T={T} three_way={three_way} eta={eta}: worst error / bound {worst:.3g}")


@pytest.mark.parametrize("three_way", [False, True])
@pytest.mark.parametrize("reproducible", [False, True])
def test_update_frames_equal_scalars_is_ddim_update(three_way, reproducible):
    from viewcrafter_b200 import ops
    prev = ops.set_reproducible(reproducible)
    try:
        for T, eta, rescale in ((25, 1.0, 0.7), (16, 0.0, 0.0), (128, 1.0, 0.7)):
            shape = (1, 4, T, 9, 16)
            x, vc, vu, vi, nz = (t.cuda() for t in _inputs(shape, 7 + T))
            kw = dict(v_uncond_img=vi, cfg_img=CFG_IMG) if three_way else {}
            for step in _frames(4, eta, True, three_way):          # includes the a = 0 step
                sc = dict(step, cfg_scale=CFG, guidance_rescale=rescale)
                a = ops.ddim_update(x, vc, vu, nz, sc, **kw)
                b = ops.ddim_update_frames(x, vc, vu, nz, sc, [step] * T, **kw)
                assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), (T, eta, rescale)
    finally:
        ops.set_reproducible(prev)


def test_update_frames_rejects_arguments():
    from viewcrafter_b200 import ops
    x = torch.zeros((1, 4, 129, 2, 2), device="cuda")
    fm = _frames(1, 1.0, True)[0]
    with pytest.raises(ops.VcError, match="T=129"):
        ops.ddim_update_frames(x, x, None, x, dict(cfg_scale=1.0, guidance_rescale=0.0), [fm] * 129)
    x4 = torch.zeros((1, 4, 4, 2, 2), device="cuda")
    with pytest.raises(ops.VcError, match="one entry of `frames` per frame"):
        ops.ddim_update_frames(x4, x4, None, x4, dict(cfg_scale=1.0, guidance_rescale=0.0), [fm] * 3)


# ------------------------------------------------------------------------------------------------ U-Net
def _unet(seed):
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
    sd = synth.synth_state_dict(synth.module_shapes(m), seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


def _err(y, ref, what):
    err = (y.cpu() - ref).abs()
    print(f"{what}: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g}")
    assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR


@pytest.mark.parametrize("mode", ["eager", "graph", "fp8", "reproducible"])
def test_unet_equal_frame_timesteps_are_the_batch_timesteps(mode):
    from viewcrafter_b200 import ops
    m, _ = _unet(21)
    g = torch.Generator().manual_seed(22)
    T = 16
    x1 = torch.randn(1, 8, T, 8, 8, generator=g)
    x, ctx = torch.cat([x1, x1], 0).cuda(), torch.randn(2, 333, 1024, generator=g).cuda()
    t, fs = torch.tensor([600, 600]).cuda(), torch.full((2,), 10).cuda()
    prev = ops.set_reproducible(mode == "reproducible")
    try:
        m.enable_fp8(mode == "fp8")
        m.enable_cuda_graph(mode == "graph")
        for shared in (False, True):
            kw = dict(cfg_shared_prefix=True) if shared else {}
            for _ in range(3 if mode == "graph" else 1):                 # eager, capture, replay
                a = m(x, t, context=ctx, fs=fs, **kw)
                b = m(x, t[:, None].repeat(1, T), context=ctx, fs=fs, **kw)
                assert torch.equal(a, b), (mode, shared)
        if mode == "graph":
            assert {k[2] for k in m._graphs} == {1, 2}                   # [B] and [B, T] are captured separately
    finally:
        m.enable_cuda_graph(False).enable_fp8(False)
        ops.set_reproducible(prev)


def _oracle(sd, *args):
    torch.set_num_threads(max(1, min(os.cpu_count() or 1, 16)))
    with torch.no_grad():
        return fr.unet_forward_frames(sd, *args)


@pytest.mark.parametrize("T", [16, 25])
def test_unet_per_frame_timesteps_shared_prefix_vs_oracle_and_graph(T):
    m, sd = _unet(23)
    g = torch.Generator().manual_seed(24)
    x1 = torch.randn(1, 8, T, 8, 8, generator=g)
    ctx = torch.randn(2, 333, 1024, generator=g)
    t1 = torch.linspace(999, 19, T).round().long()[None]
    t, fs = torch.cat([t1, t1], 0), torch.tensor([10, 10])
    ref = _oracle(sd, torch.cat([x1, x1], 0), t, ctx, fs)
    x, cc, tg, fsg = torch.cat([x1, x1], 0).cuda(), ctx.cuda(), t.cuda(), fs.cuda()
    eager = m(x, tg, context=cc, fs=fsg, cfg_shared_prefix=True)
    _err(eager, ref, f"T={T} per-frame timesteps, shared prefix")
    m.enable_cuda_graph()
    for _ in range(3):
        assert torch.equal(m(x, tg, context=cc, fs=fsg, cfg_shared_prefix=True), eager)
    flat = m(x, tg[:, :1].squeeze(1), context=cc, fs=fsg, cfg_shared_prefix=True)      # [B] recaptures, no reuse of the [B, T] graph
    assert not torch.equal(flat, eager)
    assert torch.equal(m(x, tg, context=cc, fs=fsg, cfg_shared_prefix=True), eager)
    m.enable_cuda_graph(False)


def test_unet_per_frame_timesteps_and_tokens_batch2_vs_oracle():
    m, sd = _unet(25)
    g = torch.Generator().manual_seed(26)
    T = 25
    x, ctx = torch.randn(2, 8, T, 8, 8, generator=g), torch.randn(2, 77 + 16 * T, 1024, generator=g)
    t = torch.stack([torch.linspace(999, 19, T), torch.linspace(0, 980, T)]).round().long()
    fs = torch.tensor([10, 7])
    ref = _oracle(sd, x, t, ctx, fs)
    _err(m(x.cuda(), t.cuda(), context=ctx.cuda(), fs=fs.cuda()), ref, "T=25 per-frame timesteps and tokens, B=2")


# ------------------------------------------------------------------------------------------------ the diagonal schedule is DDIM's
class FrameGaussian(_Sched):
    """The optimal denoiser for x0 ~ N(0.5, 0.8^2) (tests/test_dpm_solver_cpu.py), applied to every frame at its own timestep."""
    MU, S0 = 0.5, 0.8

    def __init__(self):
        super().__init__(dynamic=False)
        for k, v in vars(self).items():
            if isinstance(v, torch.Tensor):
                setattr(self, k, v.cuda())
        self.ac64 = self.alphas_cumprod.double()

    def apply_model(self, x, t, cond, **kwargs):
        B, T = x.shape[0], x.shape[2]
        a = self.ac64[t.reshape(B, -1).expand(B, T)].view(B, 1, T, 1, 1)
        xd = x.double()
        x0 = self.MU + a.sqrt() * self.S0 ** 2 / (a * self.S0 ** 2 + 1 - a) * (xd - a.sqrt() * self.MU)
        return ((a.sqrt() * xd - x0) / (1 - a).sqrt()).float()


@pytest.mark.parametrize("S,f,eta", [(8, 4, 1.0), (6, 2, 0.0), (4, 4, 1.0)])
def test_diagonal_schedule_is_ddim_per_frame(S, f, eta):
    """With a frame-local model and the real kernels, every output frame is its own DDIM trajectory: a frame that entered at the tail
    runs S steps from the noise it entered with, on the step noises FIFO drew for it; a frame of the initial queue runs the steps from
    its queue index k down to 0 from its queue latent."""
    from viewcrafter_b200 import ddim, fifo, ops
    model = FrameGaussian()
    B, N, h, w = 1, 3 * f + 1, 4, 6
    cc = torch.zeros(B, 4, N, h, w, device="cuda")
    cond = {"c_crossattn": [torch.zeros(B, 3, 8, device="cuda")], "c_concat": [cc]}
    kw = dict(S=S, batch_size=B, conditioning=cond, eta=eta, timestep_spacing="uniform_trailing", verbose=False)
    torch.manual_seed(11)
    out, _ = fifo.FIFOSampler(model).sample(shape=(4, N, h, w), fifo_window=f, **kw)

    # replay the draws: the warm start, the queue noise, then per iteration one noise per window and the tail frame
    smp = ddim.DDIMSampler(model)
    torch.manual_seed(11)
    z, _ = smp.sample(shape=(4, f, h, w), **dict(kw, conditioning=dict(cond, c_concat=[cc[:, :, :f]])))
    steps = [int(t) for t in smp.ddim_timesteps]
    eps = torch.randn((B, 4, S, h, w), device="cuda")
    win_noise, tail = [], []
    for m in range(N + S - f):
        win_noise.append([torch.randn((B, 4, f, h, w), device="cuda") for _ in range(S // f)])
        tail.append(torch.randn((B, 4, 1, h, w), device="cuda"))

    def ddim_from(x, k_top, noise_at):
        """DDIM steps index k_top .. 0 with ops.ddim_update on one frame [B, 4, 1, h, w]."""
        for k in range(k_top, -1, -1):
            t = torch.full((B,), steps[k], device="cuda")
            v = model.apply_model(x, t, None)
            x, _ = ops.ddim_update(x.contiguous(), v.contiguous(), None, noise_at(k).contiguous(),
                                   dict(smp.step_scalars(k, steps[k]), cfg_scale=1.0, guidance_rescale=0.0))
        return x

    for r in range(N):
        if r >= f:                                   # entered at position S - 1 after iteration r - f, then one step per iteration
            m0 = r - f + 1
            x_start = tail[m0 - 1]
        else:                                        # initial queue position k0 = r + S - f
            m0, k0 = 0, r + S - f
            x_start = (float(smp._sqrt_ac[steps[k0]]) * z[:, :, r:r + 1] + float(smp._sqrt_1mac[steps[k0]]) * eps[:, :, k0:k0 + 1])
        k_top = S - 1 if r >= f else r + S - f

        def noise_at(k, r=r, m0=m0, k_top=k_top):
            m = m0 + (k_top - k)
            return win_noise[m][k // f][:, :, k % f:k % f + 1]
        expect = ddim_from(x_start, k_top, noise_at)
        assert torch.equal(out[:, :, r:r + 1], expect), (S, f, eta, r)


# ------------------------------------------------------------------------------------------------ pipeline
def _pipeline_model():
    from tests.test_temporal_window_gpu import _pipeline_model as pm
    return pm()


@pytest.mark.parametrize("S_mult", [1, 2])
@pytest.mark.parametrize("three_way", [False, True])
def test_image_guided_synthesis_fifo_vs_oracle(three_way, S_mult):
    """image_guided_synthesis(fifo=f) (VAE encode, batched CFG with graph replay, FIFO queue, chunked VAE decode) against the FIFO
    restatement with the oracle U-Net and the float64 update, fed the same draws; from its second forward on, the U-Net replays its graph
    in the warm start and in the queue (where the [B, T] timesteps take a graph of their own)."""
    from oracle import lvdm_oracle as O
    from viewcrafter_b200 import ddim, ddim_multiplecond
    from viewcrafter_b200.synthesis import image_guided_synthesis
    model, sd, sdv, txt, txt_empty = _pipeline_model()
    unet = model.model.diffusion_model
    f = 4
    S, N = S_mult * f, 3 * f + 1
    g = torch.Generator().manual_seed(75)
    H, Wd = 8, 8
    videos = torch.rand(1, 3, N, 8 * H, 8 * Wd, generator=g) * 2 - 1
    shape = (1, 4, N, H, Wd)
    replays = []
    fwd = unet.forward

    def counting(*a, **k):
        before = unet.graph_replayed_launches
        y = fwd(*a, **k)
        replays.append(unet.graph_replayed_launches > before)
        return y
    unet.forward = counting
    extra = dict(multiple_cond_cfg=True, cfg_img=CFG_IMG) if three_way else {}
    torch.manual_seed(74)
    try:
        out = image_guided_synthesis(model, ["a photo"], videos.cuda(), list(shape), n_samples=1, ddim_steps=S, ddim_eta=1.0,
                                     unconditional_guidance_scale=CFG, fs=10, text_input=True, timestep_spacing="uniform_trailing",
                                     guidance_rescale=0.7, condition_index=[0], fifo=f, **extra)
    finally:
        del unet.forward
    assert out.shape == (1, 1, 3, N, 8 * H, 8 * Wd) and bool(torch.isfinite(out).all())
    n_warm, n_fifo = S, (N + S - f) * (S // f)
    assert len(replays) == n_warm + n_fifo
    # per phase: the first forward runs eagerly, the second captures and replays, every later one replays
    assert replays == [False] + [True] * (n_warm - 1) + [False] + [True] * (n_fifo - 1)

    torch.manual_seed(74)
    enc_noise = [torch.randn(1, 4, H, Wd) for _ in range(N)]
    img = videos[:, :, 0]
    ctx = lambda t, im: torch.cat([t, model.image_proj_model(model.embedder(im))], 1)
    ctx_c, ctx_u = ctx(txt, img), ctx(txt_empty, torch.zeros_like(img))
    ctx_i = ctx(txt_empty, img)
    fs = torch.tensor([10])
    torch.set_num_threads(max(1, min(os.cpu_count() or 1, 16)))
    with torch.no_grad():
        cc = O.encode_first_stage(sdv, videos, enc_noise)
    sched = O.model_schedule(base_scale=0.7)
    smp = (ddim_multiplecond.DDIMSampler if three_way else ddim.DDIMSampler)(model)
    smp.make_schedule(S, "uniform_trailing", 1.0, verbose=False)
    steps = [int(t) for t in smp.ddim_timesteps]
    draw = lambda shp: torch.randn(shp, device="cuda").cpu()

    def model_fn(x, t, cond, ccw):
        with torch.no_grad():
            return fr.unet_forward_frames(sd, torch.cat([x, ccw], 1), t, cond, fs)

    def warm():
        x_T = draw((1, 4, f, H, Wd))
        noises = [draw((1, 4, f, H, Wd)) for _ in range(S)]
        z, _ = O.ddim_sample(lambda x, t, c: model_fn(x, t, c, cc[:, :, :f]), sched, (1, 4, f, H, Wd), S, ctx_c, ctx_u, x_T, noises,
                             uncond_img=ctx_i if three_way else None, cfg_img=CFG_IMG if three_way else None,
                             fixed_prev_scale=not three_way)
        return z

    def denoise(p, x, renders, m):
        ks = range(p * f, p * f + f)
        t = torch.tensor([[steps[k] for k in ks]])
        ccw = cc[:, :, renders]
        vs = [model_fn(x, t, c_, ccw) for c_ in ([ctx_c, ctx_u] + ([ctx_i] if three_way else []))]
        noise = draw(x.shape)
        frames = [smp.step_scalars(k, steps[k]) for k in ks]
        kw = dict(v_uncond_img=vs[2], cfg_img=CFG_IMG) if three_way else {}
        return fr.ddim_update_frames_f64(x, vs[0], vs[1], noise, dict(cfg_scale=CFG, guidance_rescale=0.7), frames, **kw)[0].float()

    coef = lambda k: (float(smp._sqrt_ac[steps[k]]), float(smp._sqrt_1mac[steps[k]]))
    ref, _ = fr.fifo_loop(S, f, N, warm, denoise, draw, coef)
    with torch.no_grad():
        ref_img = O.decode_first_stage(sdv, ref)
    err = (out[:, 0].cpu() - ref_img).abs()
    first = float(err[:, :, :f].mean())
    print(f"fifo synthesis three_way={three_way} S={S} f={f} N={N}: mean err {float(err.mean()):.4g} (first {f} frames {first:.4g}) "
          f"max {float(err.max()):.4g} ref std {float(ref_img.std()):.3g}")
    # The frames of the warm start keep the bound of the ordinary pipeline tests.  Later frames were denoised next to frames that were
    # themselves denoised in earlier windows, so the fp16 U-Net's difference from the fp32 oracle compounds along the queue at CFG 7.5
    # on random weights (on the CPU double at S = f: mean error 0.013 at frame 0, 0.28 at frame 11); the clip gets three times the bound.
    scale = max(1.0, float(ref_img.std()))
    assert first < 0.05 * scale and float(err.mean()) < 0.15 * scale


def test_fifo_reproducible_batch_cfg_invariant():
    from viewcrafter_b200.synthesis import image_guided_synthesis
    model, *_ = _pipeline_model()
    f, N = 4, 9
    videos = (torch.rand(1, 3, N, 64, 64, generator=torch.Generator().manual_seed(3)) * 2 - 1).cuda()
    outs = []
    for batch_cfg in (True, False):
        torch.manual_seed(5)
        outs.append(image_guided_synthesis(model, ["a photo"], videos, [1, 4, N, 8, 8], ddim_steps=2 * f, ddim_eta=1.0,
                                           unconditional_guidance_scale=CFG, fs=10, text_input=True, timestep_spacing="uniform_trailing",
                                           guidance_rescale=0.7, condition_index=[0], fifo=f, batch_cfg=batch_cfg, reproducible=True))
    assert torch.equal(outs[0], outs[1])


def test_fifo_peak_memory_is_flat_in_the_clip_length():
    """Peak device memory at N = 2f + 1 and N = 8f differs by no more than the buffers that carry all N frames: the renders and their
    per-frame encode input, the latents, the output latents and the decoded clip (with its chunks and the stacked copy)."""
    from viewcrafter_b200.synthesis import image_guided_synthesis
    model, *_ = _pipeline_model()
    unet = model.model.diffusion_model
    f, h, w = 4, 8, 8
    peaks = {}
    for N in (2 * f + 1, 8 * f):
        videos = (torch.rand(1, 3, N, 8 * h, 8 * w, generator=torch.Generator().manual_seed(N)) * 2 - 1).cuda()
        unet.invalidate_packed()                 # both runs start without packed weights, K/V caches or graphs
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        torch.manual_seed(6)
        y = image_guided_synthesis(model, ["a photo"], videos, [1, 4, N, h, w], ddim_steps=2 * f, ddim_eta=1.0,
                                   unconditional_guidance_scale=CFG, fs=10, text_input=True, timestep_spacing="uniform_trailing",
                                   guidance_rescale=0.7, condition_index=[0], fifo=f)
        torch.cuda.synchronize()
        peaks[N] = torch.cuda.max_memory_allocated()
        del y, videos
    dN = 6 * f - 1
    video_frame, latent_frame = 3 * 64 * h * w * 4, 4 * h * w * 4
    allowed = dN * (6 * video_frame + 6 * latent_frame) + 8 * 2 ** 20
    print(f"peak memory: N={2 * f + 1}: {peaks[2 * f + 1] / 2**20:.2f} MiB, N={8 * f}: {peaks[8 * f] / 2**20:.2f} MiB, "
          f"difference {(peaks[8 * f] - peaks[2 * f + 1]) / 2**20:.2f} MiB, O(N) buffers {allowed / 2**20:.2f} MiB")
    assert peaks[8 * f] - peaks[2 * f + 1] <= allowed

