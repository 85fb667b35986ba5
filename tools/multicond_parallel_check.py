"""torchrun target: three-way classifier-free guidance on several GPUs vs one GPU (rank 0 prints).
  * one B=3 U-Net forward (cond, uncond, uncond_img: same x, t, fs and c_concat, three contexts) frame-sharded over all ranks
    vs the same forward on one GPU, eager and as a CUDA-graph replay.  VC_PEER_COMM=1 (default): NVLink peer-memory kernels,
    including layout switches fused into the producing GEMM's epilogue at B=3; VC_PEER_COMM=0: NCCL collectives;
  * (even world) one three-way DDIM step on the 2-way CFG split -- cond on the first half of the ranks, uncond + uncond_img as one
    B=2 forward on the second, each half frame-sharded -- vs the single-GPU step (one B=3 forward)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
from oracle import synth
from viewcrafter_b200 import parallel
from viewcrafter_b200.configs import UNET_PARAMS
from viewcrafter_b200.unet import UNetModel


def max_over_ranks(d):
    t = torch.tensor([float(d)], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


# ---- B=3 frame-sharded forward ----
m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
m.load_state_dict(synth.synth_state_dict(synth.module_shapes(m), 5), strict=True)
m = m.cuda().eval()
g = torch.Generator().manual_seed(6)
T, H, W = 4, 16, 16
x1 = torch.randn(1, 8, T, H, W, generator=g)
x, ctx = torch.cat([x1] * 3, 0).cuda(), torch.randn(3, 333, 1024, generator=g).cuda()
t, fs = torch.full((3,), 499, device="cuda"), torch.full((3,), 10, device="cuda")
y_single = m(x, t, context=ctx, fs=fs, cfg_shared_prefix=True)
comm = parallel.shard_model(m, dist, rank, world)
peer_mode = isinstance(comm, parallel.PeerFrameComm)
y_sharded = m(x, t, context=ctx, fs=fs, cfg_shared_prefix=True)          # the hint is ignored under frame sharding
torch.cuda.synchronize()
fused = getattr(comm, "fused_switches", 0)
d_fwd = max_over_ranks((y_sharded - y_single).abs().max())
m.enable_cuda_graph()
d_graph = 0.0
for _ in range(3):                                                        # eager, capture, replay
    yg = m(x, t, context=ctx, fs=fs, cfg_shared_prefix=True)
    torch.cuda.synchronize()
    d_graph = max(d_graph, float((yg - y_sharded).abs().max()))
m.enable_cuda_graph(False)
d_graph = max_over_ranks(d_graph)
need_fused = peer_mode and os.environ.get("VC_PEER_FUSED", "aligned") != "0"
ok = d_fwd < 0.02 and d_graph < 5e-3 and (fused > 0 or not need_fused)
if rank == 0:
    print(f"world {world}: peer kernels {peer_mode}; B=3 frame-sharded forward |sharded - single| {d_fwd:.4g}, graph replay vs eager "
          f"{d_graph:.4g}, layout switches fused into GEMM epilogues: {fused}")
m._comm = None

# ---- three-way DDIM step on the 2-way CFG split ----
if world % 2 == 0:
    from viewcrafter_b200.ddim_multiplecond import DDIMSampler
    from viewcrafter_b200.diffusion import LatentDiffusion
    with torch.device("cuda"):
        model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.3).eval()
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), 7), strict=True)
    unet._packed = None
    g = torch.Generator().manual_seed(8)
    shape = (1, 4, 5, 16, 16)
    xs, cc = torch.randn(shape, generator=g).cuda(), torch.randn(shape, generator=g).cuda()
    c, uc, ui = ({"c_crossattn": [torch.randn(1, 333, 1024, generator=g).cuda()], "c_concat": [cc]} for _ in range(3))
    ts = torch.full((1,), 599, dtype=torch.long, device="cuda")

    def step():
        smp = DDIMSampler(model, batch_cfg=True)
        smp.make_schedule(5, "uniform_trailing", 1.0, verbose=False)
        torch.manual_seed(9)
        return smp.p_sample_ddim(xs, c, ts, index=2, unconditional_guidance_scale=7.5, unconditional_conditioning=uc, cfg_img=2.0,
                                 unconditional_conditioning_img_nonetext=ui, fs=torch.tensor([10], device="cuda"), guidance_rescale=0.7)

    ref_step = step()
    parallel.shard_model(model, dist, rank, world, cfg_split=True)
    out_step = step()
    torch.cuda.synchronize()
    d_cfg = max_over_ranks(max(float((a - b).abs().max()) for a, b in zip(out_step, ref_step)))
    # world 2: B=1 + B=2 forwards against one B=3 forward on the same GPU (GroupNorm split counts differ with the batch; CFG 7.5
    # amplifies the fp16 rounding flips ~16x); world >= 4 adds frame sharding
    ok_cfg = d_cfg < (0.05 if world == 2 else 0.15)
    ok = ok and ok_cfg
    if rank == 0:
        print(f"world {world}: three-way step on the CFG split |sharded - single| {d_cfg:.4g}")
if rank == 0 and ok:
    print("MULTICOND_PARALLEL_CHECK_OK")
sys.stdout.flush()
torch.cuda.synchronize()
dist.barrier()
os._exit(0 if ok else 1)
