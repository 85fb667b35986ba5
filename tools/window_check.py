"""torchrun target: windowed temporal attention on several GPUs (rank 0 prints).
  * the frame-sharded U-Net forward with window (16, 4) at B = 2, T = 160 (beyond the 128 frames of full temporal attention; ranks own
    unequal frame counts, and each rank holds all frames of its sites) against the single-GPU forward, eager and replayed as a graph;
  * reproducible mode: 3 two-way DDIM steps with the window, frames sharded over all ranks, equal bit for bit (torch.equal on x_prev
    and pred_x0 of every step) to the single-GPU run each rank makes first;
  * reproducible mode, replica groups R = 2 (even world): image_guided_synthesis(temporal_window=(16, 4)) of two clips equal bit for
    bit to the same call on one GPU, including the rescheduled x_T, with both generators ending in the one-GPU state.
16x16 latents: the U-Net's deepest level runs at 2x2 sites, and frame sharding needs the site count of every level to divide by the
ranks of a frame group (4 at most here).
Prints WINDOW_CHECK_OK when every rank agrees."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
from oracle import synth
from viewcrafter_b200 import ddim, parallel, set_reproducible
from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG
from viewcrafter_b200.diffusion import LatentDiffusion
from viewcrafter_b200.synthesis import image_guided_synthesis
from viewcrafter_b200.unet import UNetModel

T, WINDOW = 160, (16, 4)


def agree(ok):
    f = torch.tensor([1.0 if ok else 0.0], device="cuda")
    dist.all_reduce(f, op=dist.ReduceOp.MIN)
    return bool(f.item() > 0)


def close(comm):
    if isinstance(comm, parallel.PeerFrameComm):
        dist.barrier()
        comm.close()


# ---- frame-sharded windowed forward vs one GPU ----
m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
m.load_state_dict(synth.synth_state_dict(synth.module_shapes(m), 5), strict=True)
m = m.cuda().eval().set_temporal_window(WINDOW)
g = torch.Generator().manual_seed(6)
x, ctx = torch.randn(2, 8, T, 16, 16, generator=g).cuda(), torch.randn(2, 333, 1024, generator=g).cuda()
t = torch.tensor([499, 19]).cuda()
y_single = m(x, t, context=ctx)
comm = parallel.shard_model(m, dist, rank, world)
y_sharded = m(x, t, context=ctx)
m.enable_cuda_graph()
d_graph = max(float((m(x, t, context=ctx) - y_sharded).abs().max()) for _ in range(3))      # eager, capture, replay
m.enable_cuda_graph(False)
d_single = float((y_sharded - y_single).abs().max())
# GroupNorm's shared-memory atomics sum in a run-dependent order outside reproducible mode: rounding flips, not bit-exactness
ok = agree(d_single < 0.02 and d_graph < 5e-3)
if rank == 0:
    print(f"world {world} ({type(comm).__name__}) T={T} window={WINDOW}: |sharded - single| {d_single:.4g}, |graph - eager| "
          f"{d_graph:.4g}: {ok}", flush=True)
close(comm)
del m

# ---- reproducible mode: 3 windowed DDIM steps, N GPUs vs 1, bit for bit ----
set_reproducible(True)


def build():
    with torch.device("cuda"):
        model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.7).eval()
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), 7), strict=True)
    unet._packed = None
    unet.set_temporal_window(WINDOW)
    return model


g = torch.Generator().manual_seed(8)
shape = (1, 4, T, 16, 16)
x0, cc = torch.randn(shape, generator=g).cuda(), torch.randn(shape, generator=g).cuda()
c, uc = ({"c_crossattn": [torch.randn(1, 333, 1024, generator=g).cuda()], "c_concat": [cc]} for _ in range(2))


def steps(model):
    smp = ddim.DDIMSampler(model, batch_cfg=True)
    smp.make_schedule(5, "uniform_trailing", 1.0, verbose=False)
    torch.manual_seed(9)
    xs, outs = x0, []
    for i, ts in enumerate((799, 599, 399)):
        xs, p0 = smp.p_sample_ddim(xs, c, torch.full((1,), ts, dtype=torch.long, device="cuda"), index=4 - i,
                                   unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=torch.tensor([10], device="cuda"),
                                   guidance_rescale=0.7)
        outs += [xs.clone(), p0.clone()]
    return outs


ref = steps(build())
model = build()
comm = parallel.shard_model(model, dist, rank, world, cfg_split=False)
out = steps(model)
torch.cuda.synchronize()
same = agree(all(torch.equal(a, b) for a, b in zip(out, ref)))
ok = ok and same
if rank == 0:
    print(f"world {world} reproducible frames T={T} window={WINDOW}: bit-identical to 1 GPU {same}", flush=True)
close(comm)
del model

# ---- reproducible mode: replica groups R = 2 vs one GPU ----
if world % 2 == 0:
    Tr, H, W = 49, 16, 16

    def build_ld():
        model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=dict(VAE_DDCONFIG, ch=32), embed_dim=4), base_scale=0.7)
        unet, vae = model.model.diffusion_model, model.first_stage_model
        unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), seed=91), strict=True)
        vae.load_state_dict(synth.synth_state_dict(synth.module_shapes(vae), seed=92), strict=True)
        model = model.cuda().eval()
        g = torch.Generator().manual_seed(93)
        W_img = (torch.randn(3 * 4 * 4, 256 * 8, generator=g) * 0.1).cuda()
        txt, txt_empty = torch.randn(1, 77, 1024, generator=g).cuda(), torch.randn(1, 77, 1024, generator=g).cuda()
        model.embedder = lambda img: torch.nn.functional.adaptive_avg_pool2d(img, 4).reshape(img.shape[0], 1, -1)
        model.image_proj_model = lambda e: (e @ W_img).reshape(e.shape[0], 256, 8).repeat(1, 1, 128)
        model.get_learned_conditioning = lambda prompts: torch.cat([txt_empty if p == "" else txt for p in prompts], 0)
        model.uncond_type = "empty_seq"
        return model

    def run(model, B=2):
        videos = (torch.rand(B, 3, Tr, 8 * H, 8 * W, generator=torch.Generator().manual_seed(94)) * 2 - 1).cuda()
        torch.manual_seed(95)
        y = image_guided_synthesis(model, ["a photo"] * B, videos, [B, 4, Tr, H, W], n_samples=1, ddim_steps=3, ddim_eta=1.0,
                                   unconditional_guidance_scale=7.5, fs=10, text_input=True, timestep_spacing="uniform_trailing",
                                   guidance_rescale=0.7, condition_index=[0], temporal_window=WINDOW, window_seed=2)
        torch.cuda.synchronize()
        return y, torch.cuda.get_rng_state(), torch.get_rng_state()

    ref = run(build_ld())
    model = build_ld()
    comm = parallel.shard_model(model, dist, rank, world, replicas=2)
    out = run(model)
    same = agree(all(torch.equal(a, b) for a, b in zip(out, ref)) and model.model.diffusion_model.temporal_window is None)
    ok = ok and same
    if rank == 0:
        print(f"world {world} reproducible replicas R=2 T={Tr} window={WINDOW}: bit-identical to 1 GPU (clips and generators) {same}",
              flush=True)
    close(comm)
set_reproducible(False)
if rank == 0 and ok:
    print("WINDOW_CHECK_OK")
sys.stdout.flush()
torch.cuda.synchronize()
dist.barrier()
os._exit(0 if ok else 1)
