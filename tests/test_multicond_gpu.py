"""Three-way classifier-free guidance on the GPU: the B=3 (cond, uncond, uncond_img) U-Net forward with the shared
context-free prefix, the three-way sampler driving it (CUDA-graph replay on), and -- with >= 2 GPUs -- the multi-GPU layouts
(tools/multicond_parallel_check.py under torch.distributed.run)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_ERR, MEAN_ERR = 0.02, 0.003          # the U-Net forward bounds of test_unet_gpu.py


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def test_batch3_shared_prefix_forward_vs_three_batch1_forwards_and_oracle():
    """One B=3 forward with cfg_shared_prefix against three B=1 forwards of the same model.  8x24 latents: 192 rows per frame
    (48, 12 and 3 at the lower levels), not a multiple of the 128-row GEMM tile, so tiles straddle frames and batch elements.
    Every kernel computes each batch
    element on its own; only the GroupNorm kernels pick their split count (and so their summation order) from the number of
    samples, which can flip the last fp16 bit -- hence a bound instead of bit equality."""
    _need_gpu()
    from oracle import lvdm_oracle as O
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
    sd = synth.synth_state_dict(synth.module_shapes(m), 21)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(22)
    x1 = torch.randn(1, 8, 5, 8, 24, generator=g)
    x, ctx = torch.cat([x1] * 3, 0), torch.randn(3, 333, 1024, generator=g)
    t, fs = torch.full((3,), 499), torch.full((3,), 10)
    xc, tc, cc, fc = x.cuda(), t.cuda(), ctx.cuda(), fs.cuda()
    y3 = m(xc, tc, context=cc, fs=fc, cfg_shared_prefix=True)
    y1 = torch.cat([m(xc[i:i + 1], tc[i:i + 1], context=cc[i:i + 1].contiguous(), fs=fc[i:i + 1]) for i in range(3)], 0)
    d = (y3 - y1).abs()
    print(f"B=3 shared prefix vs 3 x B=1: max |diff| {float(d.max()):.3g} (bit-identical: {torch.equal(y3, y1)}), "
          f"per branch {[float(d[i].max()) for i in range(3)]}")
    assert float(d.max()) <= MAX_ERR and float(d.mean()) <= MEAN_ERR
    with torch.no_grad():
        ref = O.unet_forward(sd, x, t, ctx, fs)
    err = (y3.cpu() - ref).abs()
    print(f"B=3 shared prefix vs fp32 oracle: max err {float(err.max()):.4g} mean {float(err.mean()):.4g}")
    assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR
    assert float((y3[0] - y3[2]).abs().mean()) > MEAN_ERR                    # the branches do differ (different contexts)


def test_three_way_sampler_three_steps_vs_oracle():
    """ddim_multiplecond.DDIMSampler.sample (S=3, eta=1, CFG 7.5, cfg_img 2.0, rescale 0.7, batch_cfg=True: one B=3 forward per
    step, replayed as a CUDA graph) with identical x_T and per-step noise on both sides; the bounds of
    test_ddim_sample_three_steps_vs_oracle.  The stacked context is built once, so one snapshot, one K/V cache and one graph serve
    every step."""
    _need_gpu()
    from oracle import lvdm_oracle as O
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.ddim_multiplecond import DDIMSampler
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.7)
    unet = model.model.diffusion_model
    sd = synth.synth_state_dict(synth.module_shapes(unet), seed=41)
    unet.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    g = torch.Generator().manual_seed(42)
    T, H, W, S = 5, 8, 8, 3
    shape = (1, 4, T, H, W)
    x_T, cc = torch.randn(shape, generator=g), torch.randn(shape, generator=g)
    ctx_c, ctx_u, ctx_i = (torch.randn(1, 333, 1024, generator=g) for _ in range(3))
    fs = torch.tensor([10])
    cc_d = cc.cuda()                                            # one c_concat tensor for all branches, as image_guided_synthesis passes it
    c, uc, ui = ({"c_crossattn": [k.cuda()], "c_concat": [cc_d]} for k in (ctx_c, ctx_u, ctx_i))
    unet.enable_cuda_graph()
    batches, inner = [], model.apply_model
    model.apply_model = lambda x, t, cond, **kw: (batches.append(x.shape[0]), inner(x, t, cond, **kw))[1]
    sampler = DDIMSampler(model, batch_cfg=True)
    torch.manual_seed(43)
    out, inter = sampler.sample(S=S, batch_size=1, shape=shape[1:], conditioning=c, eta=1.0, verbose=False, x_T=x_T.cuda(),
                                unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=fs.cuda(), cfg_img=2.0,
                                unconditional_conditioning_img_nonetext=ui, timestep_spacing="uniform_trailing", guidance_rescale=0.7)
    torch.manual_seed(43)
    noises = [torch.randn(shape, device="cuda").cpu() for _ in range(S)]
    sched = O.model_schedule(base_scale=0.7)

    def model_fn(x, t, cond):
        with torch.no_grad():
            return O.unet_forward(sd, torch.cat([x, cc], 1), t, cond, fs)

    ref, ref_inter = O.ddim_sample(model_fn, sched, shape, S, ctx_c, ctx_u, x_T, noises, fixed_prev_scale=False, uncond_img=ctx_i, cfg_img=2.0)
    err = (out.cpu() - ref).abs()
    print(f"three-way ddim S=3 batch_cfg=True: max err {float(err.max()):.4g} mean {float(err.mean()):.4g} ref std {float(ref.std()):.3g}")
    assert batches == [3] * S
    assert len(inter["x_inter"]) == len(ref_inter["x_inter"])
    assert float(err.max()) <= 0.15 and float(err.mean()) <= 0.02
    assert len(unet._canon) == 1 and len(unet._kv_caches) == 1
    assert sum(e["graph"] is not None for e in unet._graphs.values()) == 1


@pytest.mark.parametrize("peer", ["1", "0"])
def test_three_way_guidance_on_two_gpus(peer):
    """peer=1: NVLink peer-memory kernels with the layout switches fused into GEMM epilogues at B=3; peer=0: NCCL collectives."""
    world = 2
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} CUDA devices")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29534", os.path.join(ROOT, "tools", "multicond_parallel_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=800, env=dict(os.environ, VC_PEER_COMM=peer))
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "MULTICOND_PARALLEL_CHECK_OK" in r.stdout
