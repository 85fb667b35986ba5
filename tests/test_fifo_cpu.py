"""FIFO-Diffusion diagonal denoising (viewcrafter_b200.fifo) without a GPU:
  * the queue bookkeeping of FIFOSampler / FIFOSamplerMultiCond against the definition restated in tests/fifo_ref.py: render indices
    and timesteps of every window evaluation, output order, the iteration count N + S - f, the clamp of padding renders, every random
    draw in order and the generator's end state, with the updates replaced by float64 restatements;
  * N <= f is the ordinary sampler's call, torch.equal;
  * option validation before any forward, in the sampler, the U-Net's timesteps and image_guided_synthesis;
  * the host-side argument checks of vc_ddim_update_frames;
  * two gloo processes: the frame-sharded U-Net with [B, T] timesteps against the single process and the per-frame oracle."""
import pytest
import torch

from tests import fake_ops
from tests import fifo_ref as fr
from viewcrafter_b200 import ops, schedule
from viewcrafter_b200.ddim import DDIMSampler
from viewcrafter_b200.ddim_multiplecond import DDIMSampler as DDIMSamplerMultiCond
from viewcrafter_b200.fifo import FIFOSampler, FIFOSamplerMultiCond

C, H, W = 4, 3, 2


class StubModel:
    """A v-prediction model that is elementwise in every frame: v = 0.3 x - 0.2 c_concat + t / 1000 + 0.05 context[:, 0, 0], with t per
    frame for [B, T] timesteps.  Records the timesteps and the c_concat of every forward."""
    parameterization = "v"

    def __init__(self, dynamic=True):
        self.use_dynamic_rescale = dynamic
        for k, v in schedule.model_buffers(base_scale=0.7, dynamic_rescale=dynamic).items():
            setattr(self, k, v)
        self.num_timesteps = 1000
        self.calls = []

    @staticmethod
    def v(x, t, cc, ctx):
        T = x.shape[2]
        tt = t.float().reshape(t.shape[0], -1).expand(t.shape[0], T)
        return 0.3 * x.float() - 0.2 * cc + tt[:, None, :, None, None] / 1000 + 0.05 * ctx[:, 0, 0].view(-1, 1, 1, 1, 1)

    def apply_model(self, x, t, cond, **kwargs):
        cc, ctx = cond["c_concat"][0], cond["c_crossattn"][0]
        self.calls.append((t.clone(), cc[:, 0, :, 0, 0].clone()))
        return self.v(x, t, cc, ctx)


def _update_f32(fn):
    return lambda *a, **k: tuple(t.float() for t in fn(*a, **k))


@pytest.fixture
def f64_updates(monkeypatch):
    monkeypatch.setattr(ops, "ddim_update", _update_f32(fr.ddim_update_f64))
    monkeypatch.setattr(ops, "ddim_update_frames", _update_f32(fr.ddim_update_frames_f64))


def _conds(B, N, three_way, g):
    """Render latents whose channel 0 holds the render index (+ 1000 b), shared by every branch like image_guided_synthesis builds them."""
    cc = torch.randn(B, C, N, H, W, generator=g)
    cc[:, 0] = (torch.arange(N).view(1, N, 1, 1) + 1000 * torch.arange(B).view(B, 1, 1, 1)).float()
    mk = lambda: {"c_crossattn": [torch.randn(B, 5, 8, generator=g)], "c_concat": [cc]}
    c, uc, ui = mk(), mk(), mk()
    return cc, c, uc, (ui if three_way else None)


CASES = [  # (three_way, B, S, f, N, eta, guidance_rescale, spacing, batch_cfg)
    (False, 2, 6, 3, 8, 1.0, 0.7, "uniform_trailing", True),
    (False, 1, 4, 4, 9, 0.0, 0.0, "uniform", False),
    (True, 1, 6, 2, 5, 0.5, 0.7, "uniform_trailing", True),
    (True, 2, 4, 2, 7, 1.0, 0.0, "uniform_trailing", False),
]


@pytest.mark.parametrize("three_way,B,S,f,N,eta,rescale,spacing,batch_cfg", CASES)
def test_queue_against_the_restatement(f64_updates, three_way, B, S, f, N, eta, rescale, spacing, batch_cfg):
    g = torch.Generator().manual_seed(S * 10 + N)
    model = StubModel()
    cc, c, uc, ui = _conds(B, N, three_way, g)
    fs = torch.full((B,), 10)
    kw = dict(S=S, batch_size=B, shape=(C, N, H, W), conditioning=c, unconditional_conditioning=uc, unconditional_guidance_scale=7.5,
              eta=eta, guidance_rescale=rescale, timestep_spacing=spacing, fs=fs, verbose=False)
    if three_way:
        kw.update(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui)
    cls, base = (FIFOSamplerMultiCond, DDIMSamplerMultiCond) if three_way else (FIFOSampler, DDIMSampler)
    torch.manual_seed(3)
    out, inter = cls(model, batch_cfg=batch_cfg).sample(fifo_window=f, **kw)
    state = torch.get_rng_state()
    calls = model.calls

    # the restatement, with the same generator draws in the definition's order
    ref_model = StubModel()
    ref = base(ref_model)
    ref.make_schedule(S, spacing, eta, verbose=False)
    steps = [int(t) for t in ref.ddim_timesteps]
    assert len(steps) == S
    branches = [c, uc] + ([ui] if three_way else [])

    def warm():
        cut = lambda d: dict(d, c_concat=[d["c_concat"][0][:, :, :f]])
        wk = dict(kw, shape=(C, f, H, W), conditioning=cut(c), unconditional_conditioning=cut(uc))
        if three_way:
            wk["unconditional_conditioning_img_nonetext"] = cut(ui)
        return base(ref_model, batch_cfg=batch_cfg).sample(**wk)[0]

    def denoise(p, x, renders, m):
        ks = range(p * f, p * f + f)
        t = torch.tensor([steps[k] for k in ks]).repeat(B, 1)
        ccw = cc[:, :, renders]
        vs = [StubModel.v(x, t, ccw, br["c_crossattn"][0]) for br in branches]
        noise = torch.randn(x.shape)
        frames = [ref.step_scalars(k, steps[k]) for k in ks]
        sc = dict(cfg_scale=7.5, guidance_rescale=rescale)
        extra = dict(v_uncond_img=vs[2], cfg_img=2.0) if three_way else {}
        rows = [slice(b, b + 1) for b in range(B)] if rescale > 0 else [slice(0, B)]
        outs = [fr.ddim_update_frames_f64(x[r], vs[0][r], vs[1][r], noise[r], sc, frames,
                                          **{k: (v[r] if isinstance(v, torch.Tensor) else v) for k, v in extra.items()})[0].float()
                for r in rows]
        return torch.cat(outs, 0)

    coef = lambda k: (float(ref_model.sqrt_alphas_cumprod[steps[k]]), float(ref_model.sqrt_one_minus_alphas_cumprod[steps[k]]))
    torch.manual_seed(3)
    expect, log = fr.fifo_loop(S, f, N, warm, denoise, lambda shape: torch.randn(shape), coef)
    assert torch.equal(torch.get_rng_state(), state)
    assert out.shape == (B, C, N, H, W) and out.dtype == torch.float32
    assert torch.equal(out, expect)
    assert torch.equal(inter["x_inter"][-1], out)

    # the window evaluations: S warm-start steps, then N + S - f iterations of S / f windows, each with its timesteps and renders
    per_step = 1 if batch_cfg else (3 if three_way else 2)
    assert len(log) == (N + S - f) * (S // f)
    assert len(calls) == per_step * (S + len(log))
    fifo_calls = calls[per_step * S:]
    for i, (m, p, renders) in enumerate(log):
        assert renders == [min(max(m + k - (S - f), 0), N - 1) for k in range(p * f, p * f + f)]
        for t, ids in fifo_calls[per_step * i:per_step * (i + 1)]:
            assert t.shape == (ids.shape[0], f) and bool((t == torch.tensor(steps[p * f:p * f + f])).all())
            assert torch.equal(ids % 1000, torch.tensor(renders, dtype=torch.float32).expand_as(ids))
    # the padding renders: the head clamps to render 0 before the first output, the tail to N - 1 near the end
    assert log[0][2][0] == 0 and log[-1][2][-1] == N - 1


def test_window_timesteps_of_the_last_partition_reach_the_top():
    """Under zero-terminal SNR the tail position S - 1 is pure noise: sqrt(a(tau_{S-1})) = 0."""
    smp = DDIMSampler(StubModel())
    smp.make_schedule(50, "uniform_trailing", 1.0, verbose=False)
    assert int(smp.ddim_timesteps[-1]) == 999 and float(smp._sqrt_ac[999]) == 0.0


@pytest.mark.parametrize("three_way", [False, True])
def test_up_to_one_window_is_the_ordinary_sampler(f64_updates, three_way):
    g = torch.Generator().manual_seed(9)
    for N in (2, 4):
        cc, c, uc, ui = _conds(1, N, three_way, g)
        kw = dict(S=4, batch_size=1, shape=(C, N, H, W), conditioning=c, unconditional_conditioning=uc, unconditional_guidance_scale=7.5,
                  eta=1.0, guidance_rescale=0.7, timestep_spacing="uniform_trailing", verbose=False)
        if three_way:
            kw.update(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui)
        cls, base = (FIFOSamplerMultiCond, DDIMSamplerMultiCond) if three_way else (FIFOSampler, DDIMSampler)
        torch.manual_seed(5)
        a, ia = cls(StubModel(), batch_cfg=True).sample(fifo_window=4, **kw)
        sa = torch.get_rng_state()
        torch.manual_seed(5)
        b, ib = base(StubModel(), batch_cfg=True).sample(**kw)
        assert torch.equal(a, b) and torch.equal(sa, torch.get_rng_state())
        assert all(torch.equal(x, y) for x, y in zip(ia["x_inter"], ib["x_inter"]))


def _sample_kw(**over):
    g = torch.Generator().manual_seed(1)
    cc, c, uc, _ = _conds(1, 9, False, g)
    return dict(dict(S=4, batch_size=1, shape=(C, 9, H, W), conditioning=c, unconditional_conditioning=uc,
                     unconditional_guidance_scale=7.5, verbose=False), **over)


@pytest.mark.parametrize("window,steps", [(3, 4), (8, 4), (1, 4), (0, 4), (129, 129), (2.0, 4), (True, 4), (None, 4), ("2", 4)])
def test_bad_windows_raise_before_any_forward(window, steps):
    model = StubModel()
    with pytest.raises(ValueError, match="FIFO"):
        FIFOSampler(model).sample(fifo_window=window, **_sample_kw(S=steps))
    assert model.calls == []


@pytest.mark.parametrize("name,value", [("mask", torch.ones(1)), ("x0", torch.ones(1)), ("x_T", torch.ones(1)), ("timesteps", 3),
                                        ("noise_dropout", 0.1), ("temperature", 0.9), ("repeat_noise", True),
                                        ("score_corrector", object()), ("quantize_x0", True)])
@pytest.mark.parametrize("cls", [FIFOSampler, FIFOSamplerMultiCond])
def test_rejected_options_raise_before_any_forward(cls, name, value):
    model = StubModel()
    with pytest.raises(NotImplementedError, match=name):
        cls(model).sample(fifo_window=2, **_sample_kw(**{name: value}))
    assert model.calls == []


def test_decode_and_bad_shapes_are_rejected():
    model = StubModel()
    with pytest.raises(NotImplementedError, match="decode"):
        FIFOSampler(model).decode(None, None, 1)
    with pytest.raises(ValueError, match="shape"):
        FIFOSampler(model).sample(fifo_window=2, **_sample_kw(shape=(C, H, W)))
    kw = _sample_kw()
    kw["conditioning"] = dict(kw["conditioning"], c_concat=[kw["conditioning"]["c_concat"][0][:, :, :5]])
    with pytest.raises(ValueError, match="all 9 frames"):
        FIFOSampler(model).sample(fifo_window=2, **kw)


def test_synthesis_validates_fifo_first():
    from viewcrafter_b200.synthesis import image_guided_synthesis
    shape = [1, 4, 49, 8, 8]
    for kw, msg in ((dict(fifo=25, sampler="dpmpp_2m", ddim_eta=1.0), "sampler='ddim'"), (dict(fifo=25, temporal_window=(16, 4)), "temporal_window"),
                    (dict(fifo=7, ddim_steps=50), "multiple of the window"), (dict(fifo=1), "2 <= f"), (dict(fifo=200), "2 <= f")):
        with pytest.raises(ValueError, match=msg):
            image_guided_synthesis(None, [""], None, shape, **kw)
    replicated = type("M", (), {"_replicas": object()})()
    with pytest.raises(ValueError, match="replica"):
        image_guided_synthesis(replicated, [""], None, shape, fifo=25)


def _small_unet():
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
    sd = synth.synth_state_dict(synth.module_shapes(m), 3)
    m.load_state_dict(sd, strict=True)
    return m.eval(), sd


def test_unet_timesteps_shapes(monkeypatch):
    """[B] and [B, T] run; any other shape raises ValueError before any work.  On the CPU double, [B, T] with equal timesteps is the [B]
    forward up to the double's rounding and distinct ones match the per-frame oracle."""
    fake_ops.install(monkeypatch)
    m, sd = _small_unet()
    g = torch.Generator().manual_seed(4)
    B, T = 2, 5
    x, ctx = torch.randn(B, 8, T, 8, 8, generator=g), torch.randn(B, 333, 1024, generator=g)
    for bad in (torch.tensor([500]), torch.full((B, T + 1), 500), torch.full((B, T, 1), 500), torch.tensor(500), torch.full((T, B), 500)):
        with pytest.raises(ValueError, match="timesteps"):
            m(x, bad, context=ctx)
    t = torch.tensor([700, 30])
    # (bit-identity is the GPU test's: the double's CPU matmuls are not row-count invariant)
    assert float((m(x, t[:, None].repeat(1, T), context=ctx) - m(x, t, context=ctx)).abs().max()) < 0.02
    tf = torch.tensor([[999, 800, 600, 400, 200], [19, 39, 59, 79, 99]])
    y = m(x, tf, context=ctx)
    with torch.no_grad():
        ref = fr.unet_forward_frames(sd, x, tf, ctx)
    assert float((y - ref).abs().max()) < 0.05
    assert not torch.equal(y, m(x, t, context=ctx))


def test_graph_key_includes_the_timesteps_rank():
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
    m._forward_impl = lambda *a, **k: None
    ctx = torch.zeros(1, 4)
    for t in (torch.zeros(1), torch.zeros(1, 3)):
        m._forward_graphed(torch.zeros(1, 8, 3, 8, 8), t, ctx, None, {})
    assert len(m._graphs) == 2 and sorted(k[2] for k in m._graphs) == [1, 2]


def test_c_entry_point_rejects_arguments_before_launch():
    """vc_ddim_update_frames checks its arguments on the host, before any CUDA call."""
    import ctypes as C_
    from viewcrafter_b200 import _lib
    lib = _lib.load()
    p = 4096
    s = _lib.DdimScalars(cfg_scale=7.5, guidance_rescale=0.0, use_cfg=1)
    tab = (_lib.DdimFrameScalars * 129)()
    cases = [((p, p, p, None, 0.0, p, p, p, 4 * 16 * 8, 0, 8), tab, s, b"T=0 unsupported (1..128)"),
             ((p, p, p, None, 0.0, p, p, p, 4 * 129 * 8, 129, 8), tab, s, b"T=129 unsupported (1..128)"),
             ((p, p, p, None, 0.0, p, p, p, 4 * 16 * 8 + 8, 16, 8), tab, s, b"not a multiple of T*HW=128"),
             ((p, p, p, None, 0.0, p, p, p, 4 * 16 * 8, 16, 0), tab, s, b"not a multiple of T*HW=0"),
             ((None, p, p, None, 0.0, p, p, p, 4 * 16 * 8, 16, 8), tab, s, b"null pointer"),
             ((p, p, p, None, 0.0, p, p, p, 4 * 16 * 8, 16, 8), None, s, b"null pointer"),
             ((p, p, p, None, 0.0, p, p, p, 4 * 16 * 8, 16, 8), tab, None, b"null scalars"),
             ((p, p, None, None, 0.0, p, p, p, 4 * 16 * 8, 16, 8), tab, s, b"CFG needs the unconditional output")]
    for args, frames, sc, msg in cases:
        rc = lib.vc_ddim_update_frames(*args, C_.byref(sc) if sc is not None else None, frames, p, None)
        assert rc != 0 and msg in lib.vc_last_error(), (args, lib.vc_last_error())
    s.use_cfg = 0
    rc = lib.vc_ddim_update_frames(p, p, None, p, 2.0, p, p, p, 4 * 16 * 8, 16, 8, C_.byref(s), tab, p, None)
    assert rc != 0 and b"only defined with CFG on" in lib.vc_last_error()


def test_python_wrapper_rejects_bad_frames():
    frames = [dict(sqrt_ac_t=1.0, sqrt_1mac_t=0.0, a_prev=1.0, sigma_t=0.0, scale_t=1.0, prev_scale_t=1.0)]
    x = torch.zeros(1, 4, 2, 2, 2)
    with pytest.raises(AssertionError):                     # CPU tensors never reach the library
        ops.ddim_update_frames(x, x, None, x, dict(cfg_scale=1.0, guidance_rescale=0.0), frames * 2)


# ---- two processes (gloo) on the CPU double ----
def _gloo_worker(rank, world, port, q):
    import os
    import _pytest.monkeypatch as mpatch
    import torch.distributed as dist
    from viewcrafter_b200 import parallel
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    mpx = mpatch.MonkeyPatch()
    fake_ops.install(mpx)
    m, sd = _small_unet()
    g = torch.Generator().manual_seed(6)
    T, H_, W_ = 12, 8, 32
    x, ctx = torch.randn(2, 8, T, H_, W_, generator=g), torch.randn(2, 77 + 16 * T, 1024, generator=g)
    t = torch.randint(0, 1000, (2, T), generator=g)
    single = m(x, t, context=ctx)
    parallel.shard_model(m, dist, rank, world)
    sharded = m(x, t, context=ctx)
    res = {"d_single": float((sharded - single).abs().max())}
    if rank == 0:
        with torch.no_grad():
            res["d_ref"] = float((sharded - fr.unet_forward_frames(sd, x, t, ctx)).abs().max())
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()
    mpx.undo()


def test_frame_sharded_per_frame_timesteps_on_two_processes():
    """Two gloo ranks on the CPU double: the frame-sharded U-Net with [B, T] timesteps and per-frame image tokens (each rank takes the
    embedding rows of its frames) matches the single process and the per-frame oracle."""
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=900)
        assert p.exitcode == 0, f"rank exited with {p.exitcode}"
    res = dict(q.get(timeout=10) for _ in range(2))
    for rank in (0, 1):
        assert res[rank]["d_single"] < 0.02, res[rank]
    assert res[0]["d_ref"] < 0.05, res[0]
