"""Replica groups on the GPU (parallel.shard_model(replicas=R), synthesis.image_guided_synthesis): in reproducible mode, every group's
jobs run here in one process, group after group, and the outputs and generator states are torch.equal to the sequential call, for
two clips and two samples with two- and three-way guidance.  The model_channels=64 U-Net at 25x40x64 and the full-width one (2 steps),
both with the full-width VAE; and tools/replica_check.py under torch.distributed.run when two or more devices are present."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, H, W = 25, 40, 64


@pytest.fixture(autouse=True)
def _reproducible():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import set_reproducible
    prev = set_reproducible(True)
    yield
    set_reproducible(prev)


def _model(mc):
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=mc), dict(ddconfig=VAE_DDCONFIG, embed_dim=4), base_scale=0.7)
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), seed=91), strict=True)
    vae = model.first_stage_model
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


def _one_process_replicas(index, count, store):
    """Replicas for group `index` of `count` in this one process: gather_jobs keeps this group's job latents in `store` and returns
    every job stored so far (zeros for the groups still to run), so the last group's call returns the complete output."""
    from viewcrafter_b200 import parallel

    class OneProcess(parallel.Replicas):
        def gather_jobs(self, mine, n_jobs, shape, device):
            assert len(mine) == len(self.jobs(n_jobs))
            store.update({j: t[0].float() for j, t in zip(self.jobs(n_jobs), mine)})
            return torch.stack([store.get(j, torch.zeros(shape, device=device)) for j in range(n_jobs)])
    return OneProcess(None, index, count, count)


@pytest.mark.parametrize("mc,steps", [(64, 3), (320, 2)])
@pytest.mark.parametrize("three_way", [False, True])
def test_every_groups_jobs_match_the_sequential_call(mc, steps, three_way):
    from viewcrafter_b200.synthesis import image_guided_synthesis
    model = _model(mc)
    B, n = 2, 2
    videos = (torch.rand(B, 3, T, 8 * H, 8 * W, generator=torch.Generator().manual_seed(94)) * 2 - 1).cuda()
    kw = dict(n_samples=n, ddim_steps=steps, ddim_eta=1.0, unconditional_guidance_scale=7.5, cfg_img=(2.0 if three_way else None), fs=10,
              text_input=True, multiple_cond_cfg=three_way, timestep_spacing="uniform_trailing", guidance_rescale=0.7, condition_index=[0])

    def run():
        torch.manual_seed(95)
        out = image_guided_synthesis(model, ["a photo"] * B, videos, [B, 4, T, H, W], **kw)
        torch.cuda.synchronize()
        return out, torch.cuda.get_rng_state(), torch.get_rng_state()

    ref, cuda_rng, cpu_rng = run()
    for R in (3, 4):                         # R=3: group 0 runs clip 0 of sample 0 and clip 1 of sample 1
        store = {}
        for g in range(R):
            model._replicas = _one_process_replicas(g, R, store)
            out, c_rng, p_rng = run()
            assert torch.equal(c_rng, cuda_rng) and torch.equal(p_rng, cpu_rng), (R, g)
        del model._replicas
        d = float((out - ref).abs().max())
        print(f"model_channels={mc} three_way={three_way} R={R}: every group's jobs vs the sequential call: max |diff| {d:.3g}")
        assert out.shape == ref.shape == (B, n, 3, T, 8 * H, 8 * W) and out.dtype == ref.dtype
        assert torch.equal(out, ref), (R, d)


def test_replicas_on_several_gpus():
    """tools/replica_check.py under torch.distributed.run on two GPUs: R=2 against one GPU."""
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} CUDA devices")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29553", os.path.join(ROOT, "tools", "replica_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode == 0 and "REPLICA_CHECK_OK" in r.stdout
