"""Windowed temporal attention and noise rescheduling (FreeNoise) without a GPU: the window starts, blend weights and their sums as
the kernel computes them (`viewcrafter_b200.temporal_window`) against the definition restated in `tests/window_ref.py`; the
rescheduling against an independent restatement; option validation in Python and in the C entry point; the U-Net's dispatch and the
CUDA-graph key on the CPU double of the ops."""
import pytest
import torch

from tests import fake_ops
from tests import window_ref as wr
from viewcrafter_b200 import ops
from viewcrafter_b200 import temporal_window as tw

GRID = [(T, W, S) for W in (2, 3, 16, 25, 32) for S in sorted({1, 2, 3, 4, 7, W // 2 or 1, W}) if S <= W
        for T in sorted({1, 2, W - 1, W, W + 1, W + 2, W + S, W + S + 1, 49, 64, 129, 160, 346}) if T >= 1]


@pytest.mark.parametrize("T,W,S", GRID)
def test_window_starts_cover_every_frame(T, W, S):
    st = tw.window_starts(T, W, S)
    assert st == wr.starts(T, W, S)
    assert st == sorted(set(st)) and st[0] == 0
    if T <= W:
        assert st == [0]
        return
    assert st[-1] == T - W and all(b - a <= S for a, b in zip(st, st[1:]))
    assert all(s % S == 0 for s in st[:-1]) and all(s + W < T for s in st[:-1])
    cover = [0] * T
    for s in st:
        for t in range(s, s + W):
            cover[t] += 1
    assert min(cover) >= 1


@pytest.mark.parametrize("T,W,S", [c for c in GRID if c[0] > c[1]])
def test_weight_sums_closed_form(T, W, S):
    assert wr.weights(W) == [min(j + 1, W - j) for j in range(W)] and min(wr.weights(W)) == 1
    brute = wr.weight_sums(T, W, S)
    assert [tw.weight_sum(t, T, W, S) for t in range(T)] == brute
    assert min(brute) >= 1


def test_weights_examples():
    assert wr.weights(4) == [1, 2, 2, 1] and wr.weights(5) == [1, 2, 3, 2, 1]
    # T = 6, W = 4, S = 2: windows 0 and 2 (2 + 4 = 6 is not < 6, so the last start T - W = 2 is already the second window)
    assert tw.window_starts(6, 4, 2) == [0, 2]
    assert [tw.weight_sum(t, 6, 4, 2) for t in range(6)] == [1, 2, 3, 3, 2, 1]
    # T = 7, W = 4, S = 2: regular starts 0, 2 and the last one at 3
    assert tw.window_starts(7, 4, 2) == [0, 2, 3]
    assert [tw.weight_sum(t, 7, 4, 2) for t in range(7)] == [1, 2, 3, 4, 4, 3, 1]


@pytest.mark.parametrize("T,W,S", [(49, 25, 4), (50, 16, 4), (47, 16, 5), (33, 16, 16), (40, 8, 1), (16, 16, 4), (10, 16, 4), (30, 4, 3)])
def test_reschedule_matches_restatement(T, W, S):
    g = torch.Generator().manual_seed(T * 100 + W)
    x = torch.randn(2, 4, T, 3, 5, generator=g)
    before = torch.get_rng_state()
    y = tw.reschedule_noise(x, (W, S), seed=7)
    assert torch.equal(torch.get_rng_state(), before)
    assert torch.equal(y, wr.reschedule(x, W, S, seed=7))
    assert torch.equal(y[:, :, :W], x[:, :, :W])
    # every frame's noise is some earlier frame's original noise; rows share one schedule
    for t in range(T):
        assert any(torch.equal(y[:, :, t], x[:, :, u]) for u in range(min(t + 1, W)))
    for b in range(2):
        assert torch.equal(tw.reschedule_noise(x[b:b + 1], (W, S), seed=7), y[b:b + 1])


def test_reschedule_chains_and_truncates():
    """Frame i takes frame i - W + perm: with S = W the sources of the second chunk are frames that were themselves rescheduled,
    and a last chunk shorter than S takes the head of its permutation."""
    W, S, T = 4, 4, 14
    x = torch.arange(T, dtype=torch.float32).view(1, 1, T, 1, 1)
    y = tw.reschedule_noise(x, (W, S), seed=0).flatten().long().tolist()
    g = torch.Generator().manual_seed(0)
    p1, p2, p3 = (torch.randperm(S, generator=g).tolist() for _ in range(3))
    expect = list(range(4)) + [p1[j] for j in range(4)]
    expect += [expect[4 + p2[j]] for j in range(4)]
    expect += [expect[8 + p3[j]] for j in range(2)]
    assert y == expect
    assert sorted(y[4:8]) == [0, 1, 2, 3]


def test_reschedule_leaves_generators_alone():
    x = torch.randn(1, 4, 40, 2, 2)
    torch.manual_seed(1)
    a = torch.randn(3)
    torch.manual_seed(1)
    tw.reschedule_noise(x, (16, 4), seed=123)
    assert torch.equal(torch.randn(3), a)


@pytest.mark.parametrize("bad", [(1, 1), (33, 4), (16, 0), (16, 17), (16,), (16, 4, 1), 16, "16,4", (16.0, 4), (True, 1), (16, None)])
def test_window_validation(bad):
    with pytest.raises(ValueError, match="temporal window"):
        tw.check_window(bad)


def test_window_validation_accepts():
    assert tw.check_window(None) is None
    assert tw.check_window([25, 4]) == (25, 4) and tw.check_window((2, 1)) == (2, 1) and tw.check_window((32, 32)) == (32, 32)


def test_c_entry_point_rejects_arguments_before_launch():
    """vc_temporal_attn_windowed validates T, W, S, pitches and pointers on the host, before any CUDA call."""
    from viewcrafter_b200 import _lib
    lib = _lib.load()
    p = 4096
    cases = [((p, p, p, 64, p, 64, 0, 2, 1, 16, 4), b"T=0"), ((p, p, p, 64, p, 64, 40, 2, 1, 1, 1), b"W=1 unsupported (2..32)"),
             ((p, p, p, 64, p, 64, 40, 2, 1, 33, 1), b"W=33"), ((p, p, p, 64, p, 64, 40, 2, 1, 16, 0), b"S=0 unsupported (1..W=16)"),
             ((p, p, p, 64, p, 64, 40, 2, 1, 16, 17), b"S=17"), ((None, p, p, 64, p, 64, 40, 2, 1, 16, 4), b"null pointer"),
             ((p, p, p, 60, p, 64, 40, 2, 1, 16, 4), b"multiples of 8"), ((p, p, p, 64, p, 64, 40, 0, 1, 16, 4), b"sites=0")]
    for args, msg in cases:
        rc = lib.vc_temporal_attn_windowed(*args, 0.125, None)
        assert rc != 0 and msg in lib.vc_last_error(), (args, lib.vc_last_error())


# ---- U-Net host logic on the CPU double ----
def _fake_windowed(calls):
    def temporal_attn_windowed(q, k, v, T, sites, heads, W, S, scale=0.125, out=None):
        calls.append((T, sites, W, S))
        tok = lambda t: t.reshape(T, sites, -1)[:, :, :heads * 64].permute(1, 0, 2).reshape(sites, T, heads, 64).transpose(1, 2).float()
        o, _ = wr.windowed_ref(tok(q), tok(k), tok(v), W, S, scale)
        r = o.float().transpose(1, 2).reshape(sites, T, heads * 64).permute(1, 0, 2).reshape(T * sites, heads * 64).half()
        if out is not None:
            out.copy_(r)
            return out
        return r
    return temporal_attn_windowed


def _small_unet():
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
    sd = synth.synth_state_dict(synth.module_shapes(m), 3)
    m.load_state_dict(sd, strict=True)
    return m.eval(), sd


def test_unet_dispatch_and_validation(monkeypatch):
    fake_ops.install(monkeypatch)
    calls = []
    monkeypatch.setattr(ops, "temporal_attn_windowed", _fake_windowed(calls))
    m, sd = _small_unet()
    with pytest.raises(ValueError, match="2 <= W <= 32"):
        m.set_temporal_window((40, 4))
    assert m.temporal_window is None
    g = torch.Generator().manual_seed(4)
    T = 12
    x, ctx, t = torch.randn(1, 8, T, 8, 8, generator=g), torch.randn(1, 333, 1024, generator=g), torch.tensor([500])
    off = m(x, t, context=ctx)
    assert calls == []
    assert torch.equal(m.set_temporal_window((12, 4))(x, t, context=ctx), off) and calls == []      # W >= T: full attention
    on = m.set_temporal_window((6, 2))(x, t, context=ctx)
    assert calls and {(c[0], c[2], c[3]) for c in calls} == {(T, 6, 2)} and not torch.equal(on, off)
    from oracle import lvdm_oracle as O
    with torch.no_grad(), wr.oracle_window((6, 2)):
        ref = O.unet_forward(sd, x, t, ctx)
    assert float((on - ref).abs().max()) < 0.05


def test_graph_key_includes_the_window(monkeypatch):
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
    monkeypatch.setattr(m, "_forward_impl", lambda *a, **k: None)
    ctx = torch.zeros(1, 4)
    for window in (None, (16, 4), (16, 8)):
        m.set_temporal_window(window)
        m._forward_graphed(torch.zeros(1, 8, 1, 8, 8), torch.zeros(1), ctx, None, {})
    keys = list(m._graphs)
    assert len(keys) == 3 and {k[-3] for k in keys} == {None, (16, 4), (16, 8)}
    assert {k[-2] for k in keys} == {False} and {k[-1] for k in keys} == {ops.reproducible()}    # FP8 and reproducible stay last


def test_sampler_reschedules_only_drawn_x_T(monkeypatch):
    """ddim_sampling: with the U-Net's window set, a drawn x_T is rescheduled with window_seed; an explicit x_T is used as given;
    with _rng_rows each row is row b of the rescheduled batch draw."""
    from viewcrafter_b200 import ddim
    seen = []

    class Stop(Exception):
        pass

    def p_sample_ddim(self, img, *a, **k):
        seen.append(img.clone())
        raise Stop

    monkeypatch.setattr(ddim.DDIMSampler, "p_sample_ddim", p_sample_ddim)
    unet = type("U", (), {"temporal_window": (4, 2)})()
    model = type("M", (), {"model": type("D", (), {"diffusion_model": unet})(), "num_timesteps": 1000, "betas": torch.zeros(1)})()
    smp = ddim.DDIMSampler.__new__(ddim.DDIMSampler)
    smp.model, smp.ddim_timesteps = model, torch.tensor([1, 2]).numpy()
    smp._device = lambda: torch.device("cpu")
    shape = (3, 2, 11, 2, 2)
    for kw in (dict(window_seed=5), dict(window_seed=5, _rng_rows=(1, 2)), dict(x_T=torch.ones(shape))):
        torch.manual_seed(0)
        with pytest.raises(Stop):
            smp.ddim_sampling(None, shape, **kw)
    torch.manual_seed(0)
    expect = wr.reschedule(torch.randn(shape), 4, 2, seed=5)
    assert torch.equal(seen[0], expect) and torch.equal(seen[1], expect[1:2]) and torch.equal(seen[2], torch.ones(shape))


def test_synthesis_validates_window_first():
    from viewcrafter_b200.synthesis import image_guided_synthesis
    with pytest.raises(ValueError, match="temporal window"):
        image_guided_synthesis(None, [""], None, [1, 4, 49, 8, 8], temporal_window=(64, 4))


# ---- several processes (gloo) on the CPU double ----
def _gloo_worker(rank, world, port, q):
    import os
    import _pytest.monkeypatch as mpatch
    import torch.distributed as dist
    from oracle import lvdm_oracle as O
    from oracle import synth
    from viewcrafter_b200 import parallel
    from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG
    from viewcrafter_b200.diffusion import LatentDiffusion
    from viewcrafter_b200.synthesis import image_guided_synthesis
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    mpx = mpatch.MonkeyPatch()
    fake_ops.install(mpx)
    calls = []
    mpx.setattr(ops, "temporal_attn_windowed", _fake_windowed(calls))
    res = {}
    # frame sharding: every rank runs the windows over all T frames of its own sites
    m, sd = _small_unet()
    m.set_temporal_window((16, 4))
    g = torch.Generator().manual_seed(6)
    T, H, W = 40, 8, 32                                    # the deepest level (1x4) splits over 2 ranks
    x, ctx, t = torch.randn(2, 8, T, H, W, generator=g), torch.randn(2, 333, 1024, generator=g), torch.tensor([499, 19])
    single = m(x, t, context=ctx)
    calls.clear()
    parallel.shard_model(m, dist, rank, world)
    sharded = m(x, t, context=ctx)
    res["calls"] = sorted(set(calls))
    res["d_single"] = float((sharded - single).abs().max())
    if rank == 0:
        with torch.no_grad(), wr.oracle_window((16, 4)):
            res["d_ref"] = float((sharded - O.unet_forward(sd, x, t, ctx, None, default_fs=10)).abs().max())

    # replica groups R = 2 (one rank each): image_guided_synthesis with the window equals the single-process call
    def model():
        ld = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=dict(VAE_DDCONFIG, ch=32), embed_dim=4), base_scale=0.7).eval()
        ld.model.diffusion_model.load_state_dict(synth.synth_state_dict(synth.module_shapes(ld.model.diffusion_model), seed=81), strict=True)
        ld.first_stage_model.load_state_dict(synth.synth_state_dict(synth.module_shapes(ld.first_stage_model), seed=82), strict=True)
        g = torch.Generator().manual_seed(83)
        W_img, txt = torch.randn(3 * 4 * 4, 256 * 8, generator=g) * 0.1, torch.randn(2, 77, 1024, generator=g)
        ld.embedder = lambda img: torch.nn.functional.adaptive_avg_pool2d(img, 4).reshape(img.shape[0], 1, -1)
        ld.image_proj_model = lambda e: (e @ W_img).reshape(e.shape[0], 256, 8).repeat(1, 1, 128)
        ld.get_learned_conditioning = lambda prompts: torch.cat([txt[:1] if p == "" else txt[1:] for p in prompts], 0)
        ld.uncond_type = "empty_seq"
        return ld

    def run(ld):
        torch.manual_seed(85)
        videos = torch.rand(1, 3, 12, 64, 64, generator=torch.Generator().manual_seed(84)) * 2 - 1
        y = image_guided_synthesis(ld, ["a photo"], videos, [1, 4, 12, 8, 8], n_samples=2, ddim_steps=2, ddim_eta=1.0,
                                   unconditional_guidance_scale=7.5, fs=10, text_input=True, timestep_spacing="uniform_trailing",
                                   guidance_rescale=0.7, condition_index=[0], temporal_window=(8, 4), window_seed=2)
        return y, torch.get_rng_state()

    y1, rng1 = run(model())
    ld = model()
    parallel.shard_model(ld, dist, rank, world, cfg_split=False, replicas=2)
    y2, rng2 = run(ld)
    res["replicas_equal"] = bool(torch.equal(y1, y2)) and bool(torch.equal(rng1, rng2))
    res["window_restored"] = ld.model.diffusion_model.temporal_window is None
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()
    mpx.undo()


def test_frame_sharding_and_replica_groups_on_two_processes():
    """Two gloo ranks on the CPU double: the frame-sharded windowed forward at T = 40 runs the windows over all 40 frames of each
    rank's half of the sites and matches the single process and the windowed oracle; replica groups R = 2 with a window give the
    clips and the CPU generator state of the single-process image_guided_synthesis call."""
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
        r = res[rank]
        # all 40 frames of half the sites of each level: 8x32 / 2, 4x16 / 2, 2x8 / 2, 1x4 / 2
        assert r["calls"] == [(40, 2, 16, 4), (40, 8, 16, 4), (40, 32, 16, 4), (40, 128, 16, 4)], r["calls"]
        assert r["d_single"] < 0.02, r["d_single"]
        assert r["replicas_equal"] and r["window_restored"], r
    assert res[0]["d_ref"] < 0.02, res[0]["d_ref"]
