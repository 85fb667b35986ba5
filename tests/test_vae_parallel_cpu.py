"""The VAE encode and decode frame-sharded over all ranks (parallel.vae_encode / vae_decode, synthesis.get_latent_z and
image_guided_synthesis on a model sharded by shard_model), on the CPU: gloo process groups, CUDA ops replaced by the torch double
(tests/fake_ops.py).  Every worker computes the single-process result first, in the same process, then the sharded one:
  * per-frame calls (perframe_ae) give the same bits; batched calls agree to fp16 rounding (the double's GEMMs depend on the batch);
  * the CPU generator, which the posterior draws come from, ends in the single-process state;
  * world 8 with 5 frames leaves three ranks without a frame."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import synth
from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG


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
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), seed=71), strict=True)
    model.first_stage_model.load_state_dict(synth.synth_state_dict(synth.module_shapes(model.first_stage_model), seed=72), strict=True)
    g = torch.Generator().manual_seed(73)
    W_img, txt, txt_empty = torch.randn(3 * 4 * 4, 256 * 8, generator=g) * 0.1, torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)
    model.embedder = lambda img: torch.nn.functional.adaptive_avg_pool2d(img, 4).reshape(img.shape[0], 1, -1)
    model.image_proj_model = lambda e: (e @ W_img).reshape(e.shape[0], 256, 8).repeat(1, 1, 128)
    model.get_learned_conditioning = lambda prompts: torch.cat([txt_empty if p == "" else txt for p in prompts], 0)
    model.uncond_type = "empty_seq"
    return model


def _same(a, b, exact):
    # batched calls over other frame counts: the double's fp32 GEMM sums depend on the batch, and an fp16 activation that rounds the
    # other way moves an output by ~1e-3 (the GPU kernels' bound for GroupNorm summation order is 1e-2 on decoded frames)
    return torch.equal(a, b) if exact else (a.shape == b.shape and torch.allclose(a, b, rtol=0, atol=1e-2))


def _vae_worker(rank, world, port, B, T, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    import _pytest.monkeypatch as mpatch
    from tests import fake_ops
    from viewcrafter_b200 import parallel
    from viewcrafter_b200.synthesis import get_latent_z
    mpx = mpatch.MonkeyPatch()
    fake_ops.install(mpx)
    model = _model()
    g = torch.Generator().manual_seed(74)
    videos = torch.rand(B, 3, T, 64, 64, generator=g) * 2 - 1
    z = torch.randn(B, 4, T, 8, 8, generator=g)
    single = {}
    for pf in (True, False):
        model.perframe_ae = pf
        torch.manual_seed(75)
        lat = get_latent_z(model, videos)
        single[pf] = (lat, torch.get_rng_state(), model.decode_first_stage(z))
    parallel.shard_model(model, dist, rank, world)
    assert model._vae_comm.world == world and model._vae_comm.group is None
    res = {}
    for pf in (True, False):
        model.perframe_ae = pf
        torch.manual_seed(75)
        lat = get_latent_z(model, videos)
        rng = torch.get_rng_state()
        dec = parallel.vae_decode(model, z)
        lat1, rng1, dec1 = single[pf]
        res[pf] = dict(latents=_same(lat, lat1, pf), rng=torch.equal(rng, rng1), decode=_same(dec, dec1, pf),
                       shapes=(tuple(lat.shape) == tuple(lat1.shape), tuple(dec.shape) == tuple(dec1.shape), dec.dtype == dec1.dtype),
                       d_lat=float((lat - lat1).abs().max()), d_dec=float((dec - dec1).abs().max()))
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
        p.join(timeout=900)
        assert p.exitcode == 0, f"rank exited with {p.exitcode}"
    return q.get(timeout=10)


@pytest.mark.parametrize("world,B,T", [(2, 1, 5), (3, 1, 5), (8, 1, 5), (2, 2, 3), (3, 2, 3), (8, 2, 3)])
def test_sharded_vae_encode_and_decode_match_single_process(world, B, T):
    per_rank = _spawn(_vae_worker, world, B, T)
    for rank, res in enumerate(per_rank):
        for pf, r in res.items():
            print(f"world {world} B={B} T={T} rank {rank} perframe_ae={pf}: latents max |diff| {r['d_lat']:.3g}, decode {r['d_dec']:.3g}")
            assert r["shapes"] == (True, True, True), (rank, pf, r)
            assert r["latents"] and r["decode"] and r["rng"], (rank, pf, r)


def test_shares_concatenate_to_the_unsharded_calls(monkeypatch):
    """One process: the shares of every rank, concatenated, are the unsharded moments and decode (the functions need no process
    group), a rank past the last frame gets None, and the replayed sampling gives encode_first_stage's latents."""
    from tests import fake_ops
    from viewcrafter_b200 import parallel
    fake_ops.install(monkeypatch)
    model = _model()
    model.perframe_ae = True
    g = torch.Generator().manual_seed(76)
    videos = torch.rand(1, 3, 5, 64, 64, generator=g) * 2 - 1
    z = torch.randn(1, 4, 5, 8, 8, generator=g)
    frames = videos.permute(0, 2, 1, 3, 4).reshape(5, 3, 64, 64)
    moments = torch.cat([model.first_stage_model.encode(frames[i:i + 1]).parameters for i in range(5)], 0)
    dec = model.decode_first_stage(z.permute(0, 2, 1, 3, 4).reshape(5, 4, 8, 8))
    for world in (2, 3, 8):
        enc_s = [parallel.vae_encode_share(model, videos, r, world) for r in range(world)]
        dec_s = [parallel.vae_decode_share(model, z, r, world) for r in range(world)]
        assert [s is None for s in enc_s] == [f0 == f1 for f0, f1 in parallel.frame_ranges(5, world)]
        assert torch.equal(torch.cat([s for s in enc_s if s is not None]), moments)
        assert torch.equal(torch.cat([s for s in dec_s if s is not None]), dec)
    torch.manual_seed(77)
    ref = model.encode_first_stage(videos)
    torch.manual_seed(77)
    assert torch.equal(parallel.vae_latents_from_moments(model, moments, 1, 5), ref)


def _synthesis_worker(rank, world, port, multi, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    import _pytest.monkeypatch as mpatch
    from tests import fake_ops
    from viewcrafter_b200 import parallel
    from viewcrafter_b200.synthesis import image_guided_synthesis
    mpx = mpatch.MonkeyPatch()
    fake_ops.install(mpx)
    model = _model()
    T, H, W = 3, 8, 16                                     # the deepest U-Net level (1x2) splits over a 2-rank frame group
    videos = torch.rand(1, 3, T, 8 * H, 8 * W, generator=torch.Generator().manual_seed(78)) * 2 - 1
    # without batching, the 2-way CFG split on two ranks runs the single process's B=1 forwards: the whole clip is then bit-identical
    kw = dict(n_samples=2, ddim_steps=2, ddim_eta=1.0, unconditional_guidance_scale=7.5, cfg_img=(2.0 if multi else None), fs=10,
              text_input=True, multiple_cond_cfg=multi, timestep_spacing="uniform_trailing", guidance_rescale=0.7, condition_index=[0],
              batch_cfg=multi)

    def run():
        torch.manual_seed(79)
        out = image_guided_synthesis(model, ["a photo"], videos, [1, 4, T, H, W], **kw)
        return out, torch.get_rng_state()

    out1, rng1 = run()
    parallel.shard_model(model, dist, rank, world)
    out_s, rng_s = run()
    comm, model._vae_comm = model._vae_comm, None           # the same sharded U-Net with the VAE run whole on every rank
    out_u, rng_u = run()
    model._vae_comm = comm
    res = dict(vae_exact=torch.equal(out_s, out_u), rng=torch.equal(rng_s, rng1) and torch.equal(rng_u, rng1),
               exact_single=torch.equal(out_s, out1), d_single=float((out_s - out1).abs().max()), std=float(out1.std()),
               shape=tuple(out_s.shape))
    out = [None] * world
    dist.all_gather_object(out, res)
    if rank == 0:
        q.put(out)
    dist.barrier()
    dist.destroy_process_group()
    mpx.undo()


@pytest.mark.parametrize("world,multi", [(2, False), (4, True)])
def test_image_guided_synthesis_with_the_sharded_vae(world, multi):
    """world 2: two-way guidance on the CFG split; world 4: three-way guidance on the CFG split x 2-way frame sharding.  n_samples=2."""
    per_rank = _spawn(_synthesis_worker, world, multi)
    for rank, r in enumerate(per_rank):
        print(f"world {world} three_way={multi} rank {rank}: vs single process max |diff| {r['d_single']:.3g} (std {r['std']:.3g})")
        assert r["shape"] == (1, 2, 3, 3, 64, 128)
        assert r["vae_exact"] and r["rng"], (rank, r)
        if world == 2:
            assert r["exact_single"], (rank, r)
        else:                                  # the frame-sharded U-Net sums its 5-D GroupNorm statistics in another order
            assert r["d_single"] < 0.15 * max(1.0, r["std"]), (rank, r)
