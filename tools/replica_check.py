"""torchrun target: image_guided_synthesis on replica groups (parallel.shard_model(replicas=R)) vs the same call on one GPU, with the
model_channels=64 U-Net at 25x40x64 latents (3 DDIM steps) and the full-width VAE, perframe_ae (rank 0 prints).
  * every R > 1 that divides the world, two- and three-way guidance;
  * reproducible mode, two clips and n_samples 2 and 3: outputs torch.equal, and the CUDA and CPU generators end in the one-GPU state;
  * the default mode with one clip: bit-identical where the groups have one rank (R = world), elsewhere the maximum difference is printed.
Prints REPLICA_CHECK_OK when every rank agrees."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
from oracle import synth
from viewcrafter_b200 import parallel, set_reproducible
from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG
from viewcrafter_b200.diffusion import LatentDiffusion
from viewcrafter_b200.synthesis import image_guided_synthesis

T, H, W = 25, 40, 64


def build():
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=VAE_DDCONFIG, embed_dim=4), base_scale=0.7)
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


def run(model, B, n, three_way):
    videos = (torch.rand(B, 3, T, 8 * H, 8 * W, generator=torch.Generator().manual_seed(94)) * 2 - 1).cuda()
    torch.manual_seed(95)
    out = image_guided_synthesis(model, ["a photo"] * B, videos, [B, 4, T, H, W], n_samples=n, ddim_steps=3, ddim_eta=1.0,
                                 unconditional_guidance_scale=7.5, cfg_img=(2.0 if three_way else None), fs=10, text_input=True,
                                 multiple_cond_cfg=three_way, timestep_spacing="uniform_trailing", guidance_rescale=0.7, condition_index=[0])
    torch.cuda.synchronize()
    return out, torch.cuda.get_rng_state(), torch.get_rng_state()


ok = True
cases = [(True, 2, 2), (True, 2, 3), (False, 1, 2)]             # (reproducible, B, n_samples)
for R in [r for r in range(2, world + 1) if world % r == 0]:
    for repro, B, n in cases:
        set_reproducible(repro)
        for three_way in (False, True):
            ref = run(build(), B, n, three_way)
            model = build()
            comm = parallel.shard_model(model, dist, rank, world, replicas=R)
            out = run(model, B, n, three_way)
            same = all(torch.equal(a, b) for a, b in zip(out, ref)) and out[0].shape == ref[0].shape and out[0].dtype == ref[0].dtype
            gen = torch.equal(out[1], ref[1]) and torch.equal(out[2], ref[2])
            must = repro or world // R == 1
            flags = torch.tensor([float(same), float(gen)], device="cuda")
            diff = torch.tensor([float((out[0] - ref[0]).abs().max())], device="cuda")
            dist.all_reduce(flags, op=dist.ReduceOp.MIN)
            dist.all_reduce(diff, op=dist.ReduceOp.MAX)
            ok = ok and float(flags[1]) == 1.0 and (float(flags[0]) == 1.0 or not must)
            if rank == 0:
                print(f"world {world} R={R} reproducible={repro} B={B} n_samples={n} three_way={three_way}: bit-identical "
                      f"{float(flags[0]) == 1.0} (required {must}), generators {float(flags[1]) == 1.0}, max |diff| {float(diff):.3g}",
                      flush=True)
            if isinstance(comm, parallel.PeerFrameComm):
                dist.barrier()
                comm.close()
set_reproducible(False)
if rank == 0 and ok:
    print("REPLICA_CHECK_OK")
sys.stdout.flush()
torch.cuda.synchronize()
dist.barrier()
os._exit(0 if ok else 1)
