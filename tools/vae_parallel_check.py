"""torchrun target: the VAE encode and decode frame-sharded over all ranks (synthesis.get_latent_z, parallel.vae_decode on a model
sharded by parallel.shard_model) vs the same calls on one GPU, at 576x1024 x 25 frames with the full-width VAE (rank 0 prints).
  * layouts: pure frame sharding and (even world) the 2-way CFG split -- the VAE uses all ranks in both;
  * perframe_ae=True in the default mode and perframe_ae=False in reproducible mode: latents and decoded frames torch.equal;
  * the CPU generator (posterior draws) ends in the single-GPU state, the CUDA generator is untouched.
Prints VAE_PARALLEL_CHECK_OK when every rank agrees."""
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
from viewcrafter_b200.synthesis import get_latent_z

T, H, W = 25, 576, 1024


def build():
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=VAE_DDCONFIG, embed_dim=4), base_scale=0.3)
    vae = model.first_stage_model
    vae.load_state_dict(synth.synth_state_dict(synth.module_shapes(vae), seed=31), strict=True)
    return model.cuda().eval()


g = torch.Generator().manual_seed(32)
videos = (torch.rand(1, 3, T, H, W, generator=g) * 2 - 1).cuda()
z = torch.randn(1, 4, T, H // 8, W // 8, generator=g).cuda()


def run(model, decode):
    torch.manual_seed(33)
    cuda_rng = torch.cuda.get_rng_state()
    lat = get_latent_z(model, videos)
    rng = torch.get_rng_state()
    y = decode(z)
    torch.cuda.synchronize()
    return lat, rng, y, torch.equal(cuda_rng, torch.cuda.get_rng_state())


ok = True
layouts = [("frames", False)] + ([("cfg_split", True)] if world % 2 == 0 else [])
for perframe, repro in ((True, False), (False, True)):
    set_reproducible(repro)
    model = build()
    model.perframe_ae = perframe
    ref = run(model, model.decode_first_stage)
    for name, cfg_split in layouts:
        model = build()
        model.perframe_ae = perframe
        comm = parallel.shard_model(model, dist, rank, world, cfg_split=cfg_split)
        lat, rng, y, cuda_untouched = run(model, lambda zz: parallel.vae_decode(model, zz))
        same = torch.tensor([float(torch.equal(lat, ref[0]) and torch.equal(rng, ref[1]) and torch.equal(y, ref[2]) and cuda_untouched
                                   and y.dtype == ref[2].dtype)], device="cuda")
        diff = torch.tensor([float((lat - ref[0]).abs().max()), float((y - ref[2]).abs().max())], device="cuda")
        dist.all_reduce(same, op=dist.ReduceOp.MIN)
        dist.all_reduce(diff, op=dist.ReduceOp.MAX)
        ok = ok and float(same) == 1.0
        if rank == 0:
            print(f"world {world} {name} perframe_ae={perframe} reproducible={repro}: bit-identical {float(same) == 1.0}, "
                  f"max |diff| latents {float(diff[0]):.3g} decoded {float(diff[1]):.3g}", flush=True)
        if isinstance(comm, parallel.PeerFrameComm):
            dist.barrier()
            comm.close()
if rank == 0 and ok:
    print("VAE_PARALLEL_CHECK_OK")
sys.stdout.flush()
torch.cuda.synchronize()
dist.barrier()
os._exit(0 if ok else 1)
