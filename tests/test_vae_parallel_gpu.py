"""The frame-sharded VAE on the GPU (parallel.vae_encode_share / vae_decode_share / vae_latents_from_moments) with the full-width
VAE at 576x1024 x 25 frames: every rank's share of the encode moments and of the decode, computed here on one device for world
sizes 2, 4 and 8 and concatenated, against the unsharded calls; and tools/vae_parallel_check.py under torch.distributed.run when
two or more devices are present."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, H, W = 25, 576, 1024


@pytest.fixture(scope="module")
def setup():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=VAE_DDCONFIG, embed_dim=4), base_scale=0.3)
    vae = model.first_stage_model
    vae.load_state_dict(synth.synth_state_dict(synth.module_shapes(vae), seed=31), strict=True)
    model = model.cuda().eval()
    g = torch.Generator().manual_seed(32)
    videos = (torch.rand(1, 3, T, H, W, generator=g) * 2 - 1).cuda()
    z = torch.randn(1, 4, T, H // 8, W // 8, generator=g).cuda()
    return model, videos, z


def _unsharded_moments(model, videos):
    frames = videos.permute(0, 2, 1, 3, 4).reshape(T, 3, H, W)
    enc = model.first_stage_model.encode
    if model.perframe_ae:
        return torch.cat([enc(frames[i:i + 1]).parameters for i in range(T)], 0)
    return enc(frames).parameters


def _check(model, videos, z, exact):
    from viewcrafter_b200 import parallel
    moments = _unsharded_moments(model, videos)
    decoded = model.decode_first_stage(z.permute(0, 2, 1, 3, 4).reshape(T, 4, H // 8, W // 8))
    for world in (2, 4, 8):
        m = torch.cat([parallel.vae_encode_share(model, videos, r, world) for r in range(world)], 0)
        y = torch.cat([parallel.vae_decode_share(model, z, r, world) for r in range(world)], 0)
        dm, dy = float((m - moments).abs().max()), float((y - decoded).abs().max())
        print(f"perframe_ae={model.perframe_ae} world {world}: moments max |diff| {dm:.3g}, decoded frames {dy:.3g} "
              f"(decoded range {float(decoded.min()):.3g}..{float(decoded.max()):.3g})")
        if exact:
            assert torch.equal(m, moments) and torch.equal(y, decoded), (world, dm, dy)
        else:
            assert dy <= 1e-2, (world, dm, dy)
    # the replayed posterior sampling over the gathered moments gives encode_first_stage's latents and CPU generator state
    torch.manual_seed(34)
    ref = model.encode_first_stage(videos)
    rng = torch.get_rng_state()
    torch.manual_seed(34)
    lat = parallel.vae_latents_from_moments(model, moments, 1, T)
    assert torch.equal(lat, ref) and torch.equal(torch.get_rng_state(), rng)


def test_per_frame_shares_bit_identical(setup):
    """perframe_ae=True (the ViewCrafter default), default mode: every frame goes through the same N=1 call."""
    model, videos, z = setup
    model.perframe_ae = True
    _check(model, videos, z, exact=True)


def test_batched_shares_bit_identical_in_reproducible_mode(setup):
    from viewcrafter_b200 import set_reproducible
    model, videos, z = setup
    model.perframe_ae = False
    prev = set_reproducible(True)
    try:
        _check(model, videos, z, exact=True)
    finally:
        set_reproducible(prev)
        model.perframe_ae = True


def test_batched_shares_in_the_default_mode_within_1e_2(setup):
    """perframe_ae=False without reproducible mode: the GroupNorm split count follows the batch size, so the shares differ from the
    one 25-frame call by summation order only."""
    model, videos, z = setup
    model.perframe_ae = False
    try:
        _check(model, videos, z, exact=False)
    finally:
        model.perframe_ae = True


@pytest.mark.parametrize("world", [2, 8])
def test_sharded_vae_on_several_gpus(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} CUDA devices")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29547", os.path.join(ROOT, "tools", "vae_parallel_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
    print(r.stdout[-3000:], r.stderr[-2000:])
    assert r.returncode == 0 and "VAE_PARALLEL_CHECK_OK" in r.stdout
