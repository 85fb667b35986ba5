"""torchrun target: reproducible mode on several GPUs vs one GPU, bit for bit (rank 0 prints).  Run with VC_REPRODUCIBLE=1;
VC_PEER_COMM=1 (default) uses the NVLink peer-memory kernels, 0 the NCCL collectives.
  * 3 DDIM steps, two-way and three-way guidance, with the frames sharded over all ranks (eager steps, then CUDA-graph replay);
  * (even world) the same with the 2-way CFG split (each half frame-sharded over world / 2 ranks).
Every rank compares x_prev and pred_x0 of every step with torch.equal against the single-GPU run it made first."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
from oracle import synth
from viewcrafter_b200 import ddim, ddim_multiplecond, parallel, reproducible
from viewcrafter_b200.configs import UNET_PARAMS
from viewcrafter_b200.diffusion import LatentDiffusion

assert reproducible(), "run with VC_REPRODUCIBLE=1"


def build():
    with torch.device("cuda"):
        model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.7).eval()
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), 7), strict=True)
    unet._packed = None
    return model


g = torch.Generator().manual_seed(8)
shape = (1, 4, 25, 40, 64)
x0, cc = torch.randn(shape, generator=g).cuda(), torch.randn(shape, generator=g).cuda()
c, uc, ui = ({"c_crossattn": [torch.randn(1, 333, 1024, generator=g).cuda()], "c_concat": [cc]} for _ in range(3))


def steps(model, three_way, graph):
    model.model.diffusion_model.enable_cuda_graph(graph)
    smp = (ddim_multiplecond if three_way else ddim).DDIMSampler(model, batch_cfg=True)
    smp.make_schedule(5, "uniform_trailing", 1.0, verbose=False)
    kw = dict(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui) if three_way else {}
    torch.manual_seed(9)
    x, outs = x0, []
    for i, t in enumerate((799, 599, 399)):
        ts = torch.full((1,), t, dtype=torch.long, device="cuda")
        x, p0 = smp.p_sample_ddim(x, c, ts, index=4 - i, unconditional_guidance_scale=7.5, unconditional_conditioning=uc,
                                  fs=torch.tensor([10], device="cuda"), guidance_rescale=0.7, **kw)
        outs += [x.clone(), p0.clone()]
    return outs


ok = True
layouts = [("frames", False)] + ([("cfg_split", True)] if world % 2 == 0 else [])
for three_way in (False, True):
    ref = steps(build(), three_way, False)
    for name, cfg_split in layouts:
        model = build()
        comm = parallel.shard_model(model, dist, rank, world, cfg_split=cfg_split)
        for graph in (False, True):
            out = steps(model, three_way, graph)
            if graph:
                out = steps(model, three_way, graph)            # eager + capture above, replay here
            torch.cuda.synchronize()
            same = torch.tensor([float(all(torch.equal(a, b) for a, b in zip(out, ref)))], device="cuda")
            diff = torch.tensor([max(float((a - b).abs().max()) for a, b in zip(out, ref))], device="cuda")
            dist.all_reduce(same, op=dist.ReduceOp.MIN)
            dist.all_reduce(diff, op=dist.ReduceOp.MAX)
            ok = ok and float(same) == 1.0
            if rank == 0:
                print(f"world {world} {name} ({type(comm).__name__ if comm else 'no frame sharding'}) three_way={three_way} graph={graph}: "
                      f"bit-identical {float(same) == 1.0}, max |diff| {float(diff):.3g}")
        if isinstance(comm, parallel.PeerFrameComm):
            dist.barrier()
            comm.close()
if rank == 0 and ok:
    print("REPRODUCIBLE_CHECK_OK")
sys.stdout.flush()
torch.cuda.synchronize()
dist.barrier()
os._exit(0 if ok else 1)
