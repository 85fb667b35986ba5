"""Replica groups (parallel.shard_model(replicas=R)): image_guided_synthesis runs the n_samples x B outputs of one call concurrently on
R groups of world / R ranks, on the CPU: gloo process groups, CUDA ops replaced by the torch double (tests/fake_ops.py).
  * every worker computes the single-process call first, in the same process, then the replicated one; outputs are torch.equal where
    a job's computation is the single-process one (groups of one rank, one clip), elsewhere within the double's tolerance; shapes,
    dtypes and the generator end state are always torch.equal;
  * world 2 (R=2), world 4 (R=2, 4) and world 8 (R=2, 4, 8), n_samples 1, 2, 3 and 5, one and two clips, two- and three-way guidance,
    the CFG split on and off inside a group; n_samples x B < R leaves groups idle;
  * DDIMSampler.skip_sample_draws and sample(_rng_rows=...) against real sample calls, shard_model's checks, the rejected options."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import synth
from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG

T, H, W = 4, 8, 32                     # the deepest U-Net level (1x4) splits over a frame group of four ranks


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _model():
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=dict(VAE_DDCONFIG, ch=32), embed_dim=4), base_scale=0.7).eval()
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), seed=81), strict=True)
    model.first_stage_model.load_state_dict(synth.synth_state_dict(synth.module_shapes(model.first_stage_model), seed=82), strict=True)
    g = torch.Generator().manual_seed(83)
    W_img, txt, txt_empty = torch.randn(3 * 4 * 4, 256 * 8, generator=g) * 0.1, torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)
    model.embedder = lambda img: torch.nn.functional.adaptive_avg_pool2d(img, 4).reshape(img.shape[0], 1, -1)
    model.image_proj_model = lambda e: (e @ W_img).reshape(e.shape[0], 256, 8).repeat(1, 1, 128)
    model.get_learned_conditioning = lambda prompts: torch.cat([txt_empty if p == "" else txt for p in prompts], 0)
    model.uncond_type = "empty_seq"
    return model


def _videos(B):
    return torch.rand(B, 3, T, 8 * H, 8 * W, generator=torch.Generator().manual_seed(84)) * 2 - 1


def _kw(multi, n, cfg_img=2.0):
    return dict(n_samples=n, ddim_steps=2, ddim_eta=1.0, unconditional_guidance_scale=7.5, cfg_img=(cfg_img if multi else None), fs=10,
                text_input=True, multiple_cond_cfg=multi, timestep_spacing="uniform_trailing", guidance_rescale=0.7, condition_index=[0])


def _run(model, B, multi, n):
    from viewcrafter_b200.synthesis import image_guided_synthesis
    torch.manual_seed(85)
    out = image_guided_synthesis(model, ["a photo"] * B, _videos(B), [B, 4, T, H, W], **_kw(multi, n))
    return out, torch.get_rng_state()


def _worker(rank, world, port, cases, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    import _pytest.monkeypatch as mpatch
    from tests import fake_ops
    from viewcrafter_b200 import parallel
    mpx = mpatch.MonkeyPatch()
    fake_ops.install(mpx)
    res = []
    for R, cfg_split, B, multi, n in cases:
        out1, rng1 = _run(_model(), B, multi, n)
        model = _model()
        parallel.shard_model(model, dist, rank, world, cfg_split=cfg_split, replicas=R)
        reps, unet = model._replicas, model.model.diffusion_model
        G = world // R
        split = cfg_split and G % 2 == 0
        layout = (reps.index == rank // G, reps.count == R, getattr(model, "_cfg", None) is not None,
                  (unet._comm.world if unet._comm else 1), model._vae_comm.world)
        out, rng = _run(model, B, multi, n)
        res.append(dict(case=(R, cfg_split, B, multi, n), layout=layout == (True, True, split, G // 2 if split else G, world),
                        jobs=reps.jobs(n * B), shape=(out.shape == out1.shape, out.dtype == out1.dtype), rng=torch.equal(rng, rng1),
                        exact=torch.equal(out, out1), d=float((out - out1).abs().max()), std=float(out1.std())))
    out = [None] * world
    dist.all_gather_object(out, res)
    if rank == 0:
        q.put(out)
    dist.barrier()
    dist.destroy_process_group()
    mpx.undo()


def _spawn(target, world, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port) + args + (q,)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=1500)
        assert p.exitcode == 0, f"rank exited with {p.exitcode}"
    return q.get(timeout=10)


# (R, cfg_split, B, three-way guidance, n_samples) per world size
CASES = {
    2: [(2, True, 1, False, 1), (2, True, 1, True, 3), (2, True, 2, False, 2), (2, True, 2, True, 5)],
    4: [(2, True, 1, False, 2), (2, False, 2, True, 3), (2, True, 2, True, 1), (4, True, 1, True, 5), (4, True, 2, False, 1)],
    8: [(2, True, 2, True, 2), (2, False, 1, False, 3), (4, True, 1, True, 1), (4, False, 2, False, 5), (8, True, 1, False, 5),
        (8, True, 2, True, 3)],
}


@pytest.mark.parametrize("world", sorted(CASES))
def test_replicated_synthesis_matches_single_process(world):
    per_rank = _spawn(_worker, world, CASES[world])
    for rank, results in enumerate(per_rank):
        for r in results:
            R, cfg_split, B, multi, n = r["case"]
            G = world // R
            print(f"world {world} R={R} cfg_split={cfg_split} B={B} three_way={multi} n_samples={n} rank {rank}: jobs {r['jobs']}, "
                  f"vs single process max |diff| {r['d']:.3g} (std {r['std']:.3g})")
            assert r["layout"] and r["shape"] == (True, True) and r["rng"], (world, rank, r)
            assert r["jobs"] == list(range(rank // G, n * B, R)), (world, rank, r)
            if G == 1 and B == 1:                    # each job is exactly the one-process computation
                assert r["exact"], (world, rank, r)
            else:                                    # other batch sizes / frame sharding change the fp16 roundings (CFG amplifies them)
                assert r["d"] < 0.15 * max(1.0, r["std"]), (world, rank, r)
    # every world size has a call with n_samples x B < R: the idle groups' ranks have no job and only join the gathers
    assert any(not r["jobs"] for results in per_rank for r in results)


def _sampler_problem(three_way):
    from viewcrafter_b200 import ddim, ddim_multiplecond
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.7).eval()
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), seed=86), strict=True)
    g = torch.Generator().manual_seed(87)
    B, shape = 3, (4, 2, 8, 8)
    cc = torch.randn(B, *shape, generator=g)
    c, uc, ui = ({"c_crossattn": [torch.randn(B, 333, 1024, generator=g)], "c_concat": [cc]} for _ in range(3))
    base = (ddim_multiplecond if three_way else ddim).DDIMSampler

    class Recording(base):
        """Keeps every step's noise (the draws the replay must reproduce)."""
        noises = []

        @staticmethod
        def _step_noise(*a):
            out = base._step_noise(*a)
            Recording.noises.append(out)
            return out
    kw = dict(unconditional_conditioning_img_nonetext=ui, cfg_img=2.0) if three_way else {}
    kw.update(shape=shape, eta=1.0, verbose=False, unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=torch.full((B,), 10),
              guidance_rescale=0.7, conditioning=c)
    return model, Recording, B, kw


@pytest.mark.parametrize("three_way", [False, True])
def test_row_replay_against_real_sample_calls(monkeypatch, three_way):
    """sample(_rng_rows=(b, b + 1)) draws x_T and every step's noise of the whole batch and keeps row b; skip_sample_draws consumes
    what one sample() call consumes (also with 'uniform' spacing, whose schedule has 7 steps for S=6)."""
    from tests import fake_ops
    from viewcrafter_b200.synthesis import _rows
    fake_ops.install(monkeypatch)
    model, Smp, B, kw = _sampler_problem(three_way)
    for spacing, S in (("uniform_trailing", 2), ("uniform", 6)):
        torch.manual_seed(88)
        Smp.noises = []
        out, inter = Smp(model, batch_cfg=True).sample(S=S, batch_size=B, timestep_spacing=spacing, **kw)
        full_noise, end = Smp.noises, torch.get_rng_state()
        torch.manual_seed(88)
        Smp(model).skip_sample_draws(S, (B, *kw["shape"]), torch.device("cpu"), spacing)
        assert torch.equal(torch.get_rng_state(), end), spacing
        for b in range(B):
            c, u, ui = _rows((kw["conditioning"], kw["unconditional_conditioning"], kw.get("unconditional_conditioning_img_nonetext")), b)
            assert c["c_concat"][0] is u["c_concat"][0]
            kb = dict(kw, conditioning=c, unconditional_conditioning=u, fs=kw["fs"][b:b + 1])
            if three_way:
                kb["unconditional_conditioning_img_nonetext"] = ui
            torch.manual_seed(88)
            Smp.noises = []
            o, it = Smp(model, batch_cfg=True).sample(S=S, batch_size=B, timestep_spacing=spacing, _rng_rows=(b, b + 1), **kb)
            assert torch.equal(torch.get_rng_state(), end)
            assert torch.equal(it["x_inter"][0], inter["x_inter"][0][b:b + 1])                  # x_T
            assert len(Smp.noises) == len(full_noise) and all(torch.equal(a, f[b:b + 1]) for a, f in zip(Smp.noises, full_noise))
            assert o.shape == out[b:b + 1].shape and float((o - out[b:b + 1]).abs().max()) < 0.15 * max(1.0, float(out.std()))
    # the options whose draws a row cannot replay
    for bad, name in ((dict(noise_dropout=0.1), "noise_dropout"), (dict(mask=torch.ones(1), x0=torch.zeros(1)), "mask"),
                      (dict(x0=torch.zeros(1)), "x0"), (dict(x_T=torch.zeros(1)), "x_T"), (dict(timesteps=1), "timesteps"),
                      (dict(repeat_noise=True), "repeat_noise")):
        with pytest.raises(ValueError, match=name):
            Smp(model).sample(S=2, batch_size=B, _rng_rows=(0, 1), **dict(kw, **bad))


def test_replicated_synthesis_rejects_options_before_any_work(monkeypatch):
    """image_guided_synthesis on a replicated model raises ValueError for noise_dropout > 0 (and the other options check_row_replay
    names) before the encode, so every rank raises alike and no generator moves."""
    from tests import fake_ops
    from viewcrafter_b200 import parallel
    from viewcrafter_b200.synthesis import image_guided_synthesis
    fake_ops.install(monkeypatch)
    model = _model()
    model._replicas = parallel.Replicas(None, 0, 2, 2)
    torch.manual_seed(89)
    rng = torch.get_rng_state()
    for bad, name in ((dict(noise_dropout=0.5), "noise_dropout"), (dict(timesteps=1), "timesteps"), (dict(repeat_noise=True), "repeat_noise")):
        with pytest.raises(ValueError, match=name):
            image_guided_synthesis(model, ["a photo"], _videos(1), [1, 4, T, H, W], **_kw(False, 2), **bad)
    assert torch.equal(torch.get_rng_state(), rng)


def _shard_worker(rank, world, port, replicas, repro, cfg_split, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from viewcrafter_b200 import ops, parallel
    ops.set_reproducible(repro)
    try:
        parallel.shard_model(torch.nn.Linear(2, 2), dist, rank, world, cfg_split=cfg_split, replicas=replicas[rank])
        q.put("ok")
    except (ValueError, RuntimeError) as e:
        q.put(type(e).__name__ + ": " + str(e))
    dist.destroy_process_group()


def _shard(world, replicas, repro=False, cfg_split=True):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, replicas, repro, cfg_split, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    return [q.get(timeout=10) for _ in range(world)]


def test_shard_model_replica_checks():
    out = _shard(4, (3, 3, 3, 3))
    assert all(o.startswith("ValueError") and "divides the world size 4" in o for o in out), out
    out = _shard(2, (0, 0))
    assert all(o.startswith("ValueError") and "positive integer" in o for o in out), out
    out = _shard(2, (1, 2))
    assert all(o.startswith("ValueError") and "disagree on replicas" in o for o in out), out
    # reproducible mode checks the frame groups inside a replica group: 3 ranks frame-sharded fail, 3 groups of one rank do not
    out = _shard(3, (1, 1, 1), repro=True, cfg_split=False)
    assert all("frame groups of 1, 2, 4 or 8" in o for o in out), out
    assert _shard(3, (3, 3, 3), repro=True, cfg_split=False) == ["ok"] * 3
