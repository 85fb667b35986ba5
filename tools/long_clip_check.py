"""torchrun target: a 49-frame clip on several GPUs (rank 0 prints).  VC_PEER_COMM=1 (default): the NVLink peer-memory kernels,
0: NCCL collectives.
  * the frame-sharded U-Net forward (B = 2, T = 49: ranks own unequal frame counts) against the single-GPU forward, eager and
    replayed as a CUDA graph;
  * reproducible mode: 3 two-way DDIM steps with the frames sharded over all ranks, and (even world) with the 2-way CFG split, equal bit
    for bit (torch.equal on x_prev and pred_x0 of every step) to the single-GPU run each rank makes first."""
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
from viewcrafter_b200.configs import UNET_PARAMS
from viewcrafter_b200.diffusion import LatentDiffusion
from viewcrafter_b200.unet import UNetModel

T = 49


def agree(ok):
    f = torch.tensor([1.0 if ok else 0.0], device="cuda")
    dist.all_reduce(f, op=dist.ReduceOp.MIN)
    return bool(f.item() > 0)


# ---- frame-sharded forward vs one GPU ----
m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
m.load_state_dict(synth.synth_state_dict(synth.module_shapes(m), 5), strict=True)
m = m.cuda().eval()
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
    print(f"world {world} ({type(comm).__name__}) T={T}: |sharded - single| {d_single:.4g}, |graph - eager| {d_graph:.4g}: {ok}", flush=True)
if isinstance(comm, parallel.PeerFrameComm):
    dist.barrier()
    comm.close()
del m

# ---- reproducible mode: 3 DDIM steps, N GPUs vs 1, bit for bit ----
set_reproducible(True)


def build():
    with torch.device("cuda"):
        model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.7).eval()
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), 7), strict=True)
    unet._packed = None
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
for name, cfg_split in [("frames", False)] + ([("cfg_split", True)] if world % 2 == 0 else []):
    model = build()
    comm = parallel.shard_model(model, dist, rank, world, cfg_split=cfg_split)
    out = steps(model)
    torch.cuda.synchronize()
    same = agree(all(torch.equal(a, b) for a, b in zip(out, ref)))
    ok = ok and same
    if rank == 0:
        print(f"world {world} reproducible {name} T={T}: bit-identical to 1 GPU {same}", flush=True)
    if isinstance(comm, parallel.PeerFrameComm):
        dist.barrier()
        comm.close()
if rank == 0 and ok:
    print("LONG_CLIP_CHECK_OK")
sys.stdout.flush()
torch.cuda.synchronize()
dist.barrier()
os._exit(0 if ok else 1)
