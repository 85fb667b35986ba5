"""Reproducible mode on the GPU (viewcrafter_b200.set_reproducible): the same inputs give bit-identical results whatever the batching
of the guidance branches, per-frame or batched VAE calls and the SM count.  Every comparison is torch.equal."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_ERR, MEAN_ERR = 0.02, 0.003          # the U-Net forward bounds of test_unet_gpu.py


@pytest.fixture(autouse=True)
def _reproducible():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import set_reproducible
    prev = set_reproducible(True)
    yield
    set_reproducible(prev)


def _unet(mc, seed=21):
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=mc))
    sd = synth.synth_state_dict(synth.module_shapes(m), seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


def _inputs(B, T, H, W, seed=22):
    g = torch.Generator().manual_seed(seed)
    x1 = torch.randn(1, 8, T, H, W, generator=g)
    x, ctx = torch.cat([x1] * B, 0), torch.randn(B, 333, 1024, generator=g)
    return x, ctx, torch.full((B,), 499), torch.full((B,), 10)


def test_groupnorm_canonical_matches_torch_and_is_batch_invariant():
    """The leaf kernels against torch's GroupNorm, with the x1|x2 concat and an odd frame size (nc = 1), and a batch of three frames
    against the three frames one by one."""
    import torch.nn.functional as F
    from viewcrafter_b200 import ops
    g = torch.Generator().manual_seed(3)
    for hw, C1, C2 in ((2560, 320, 0), (40, 640, 640), (35, 320, 320), (9216, 128, 0)):
        x = (torch.randn(3 * hw, C1, generator=g) * 2 + 0.5).half().cuda()
        x2 = (torch.randn(3 * hw, C2, generator=g)).half().cuda() if C2 else None
        gamma, beta = torch.rand(C1 + C2, generator=g).cuda() + 0.5, torch.randn(C1 + C2, generator=g).cuda()
        y = ops.groupnorm(x, 3, gamma, beta, 1e-5, True, x2=x2)
        a = x.float() if x2 is None else torch.cat([x, x2], 1).float()
        ref = F.silu(F.group_norm(a.view(3, hw, -1).permute(0, 2, 1), 32, gamma, beta, 1e-5)).permute(0, 2, 1).reshape(3 * hw, -1)
        assert float((y.float() - ref).abs().max()) < 2e-2, (hw, C1, C2)
        one = torch.cat([ops.groupnorm(x[i * hw:(i + 1) * hw].contiguous(), 1, gamma, beta, 1e-5, True,
                                       x2=None if x2 is None else x2[i * hw:(i + 1) * hw].contiguous()) for i in range(3)], 0)
        assert torch.equal(y, one), (hw, C1, C2)
        y5 = ops.groupnorm_canonical(x, 1, hw, gamma, beta, 1e-5, False, x2=x2)       # one sample of three frames (5-D)
        ref5 = F.group_norm(a.view(1, 3 * hw, -1).permute(0, 2, 1), 32, gamma, beta, 1e-5).permute(0, 2, 1).reshape(3 * hw, -1)
        assert float((y5.float() - ref5).abs().max()) < 2e-2, (hw, C1, C2)


@pytest.mark.parametrize("mc,T", [(64, 5), (320, 25)])
def test_unet_batched_guidance_is_bit_identical_to_batch1(mc, T):
    """B=2 and B=3 forwards with the shared CFG prefix against separate B=1 forwards at 40x64 latents (per-frame tensors of the
    full-width model cross the 16 MB producer-statistics threshold; level 3 has 40-pixel frames)."""
    m, sd = _unet(mc)
    x, ctx, t, fs = _inputs(3, T, 40, 64)
    xc, tc, cc, fc = x.cuda(), t.cuda(), ctx.cuda(), fs.cuda()
    y1 = torch.cat([m(xc[i:i + 1], tc[i:i + 1], context=cc[i:i + 1].contiguous(), fs=fc[i:i + 1]) for i in range(3)], 0)
    for B in (2, 3):
        yb = m(xc[:B], tc[:B], context=cc[:B].contiguous(), fs=fc[:B], cfg_shared_prefix=True)
        d = float((yb - y1[:B]).abs().max())
        print(f"mc={mc} T={T}: B={B} shared prefix vs B=1 forwards: max |diff| {d:.3g}")
        assert torch.equal(yb, y1[:B])
    if mc == 64:
        from oracle import lvdm_oracle as O
        with torch.no_grad():
            ref = O.unet_forward(sd, x, t, ctx, fs)
        err = (y1.cpu() - ref).abs()
        print(f"reproducible mode vs fp32 oracle: max err {float(err.max()):.4g} mean {float(err.mean()):.4g}")
        assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR


def _sample(three_way, batch_cfg):
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.diffusion import LatentDiffusion
    from viewcrafter_b200 import ddim, ddim_multiplecond
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.7)
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), seed=41), strict=True)
    model = model.cuda().eval()
    unet.enable_cuda_graph()
    g = torch.Generator().manual_seed(42)
    shape = (1, 4, 5, 40, 64)
    x_T, cc = torch.randn(shape, generator=g).cuda(), torch.randn(shape, generator=g).cuda()
    c, uc, ui = ({"c_crossattn": [torch.randn(1, 333, 1024, generator=g).cuda()], "c_concat": [cc]} for _ in range(3))
    kw = dict(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui) if three_way else {}
    S = (ddim_multiplecond if three_way else ddim).DDIMSampler(model, batch_cfg=batch_cfg)
    torch.manual_seed(43)
    out, inter = S.sample(S=3, batch_size=1, shape=shape[1:], conditioning=c, eta=1.0, verbose=False, x_T=x_T,
                          unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=torch.tensor([10]).cuda(),
                          timestep_spacing="uniform_trailing", guidance_rescale=0.7, **kw)
    replays = unet.graph_replayed_launches
    return out, inter["pred_x0"][-1], replays


@pytest.mark.parametrize("three_way", [False, True])
def test_ddim_sample_batch_cfg_on_and_off_bit_identical(three_way):
    a, pa, ra = _sample(three_way, True)
    b, pb, rb = _sample(three_way, False)
    print(f"three_way={three_way}: batch_cfg on vs off: x max |diff| {float((a - b).abs().max()):.3g}, "
          f"pred_x0 {float((pa - pb).abs().max()):.3g}; graph-replayed launches {ra} / {rb}")
    assert ra > 0 and rb > 0
    assert torch.equal(a, b) and torch.equal(pa, pb)


def test_vae_per_frame_and_batched_calls_bit_identical():
    """decode per frame vs 5 frames per call at 576x1024, and the encoder's moments the same way."""
    from oracle import synth
    from viewcrafter_b200.autoencoder import AutoencoderKL
    from viewcrafter_b200.configs import VAE_DDCONFIG
    vae = AutoencoderKL(VAE_DDCONFIG, None, 4)
    vae.load_state_dict(synth.synth_state_dict(synth.module_shapes(vae), seed=31), strict=True)
    vae = vae.cuda().eval()
    g = torch.Generator().manual_seed(32)
    z = torch.randn(5, 4, 72, 128, generator=g).cuda()
    y5 = vae.decode(z)
    y1 = torch.cat([vae.decode(z[i:i + 1]) for i in range(5)], 0)
    print(f"VAE decode 5 frames vs 1 by 1: max |diff| {float((y5 - y1).abs().max()):.3g}")
    assert torch.equal(y5, y1)
    x = torch.rand(5, 3, 576, 1024, generator=g).cuda() * 2 - 1
    m5 = vae.encode_moments(x)
    m1 = torch.cat([vae.encode_moments(x[i:i + 1]) for i in range(5)], 0)
    print(f"VAE encode 5 frames vs 1 by 1: max |diff| {float((m5 - m1).abs().max()):.3g}")
    assert torch.equal(m5, m1)


_SM_SCRIPT = r"""
import os, sys
sys.path.insert(0, {root!r})
import torch
from viewcrafter_b200 import ops
from tests.test_reproducible_gpu import _unet, _inputs
m, _ = _unet(320)
x, ctx, t, fs = _inputs(2, 25, 40, 64)
y = m(x.cuda(), t.cuda(), context=ctx.cuda(), fs=fs.cuda(), cfg_shared_prefix=True)
g = torch.Generator().manual_seed(5)
xs, vc, vu, nz = (torch.randn(4 * 25 * 40 * 64, generator=g).cuda() for _ in range(4))
sc = dict(cfg_scale=7.5, guidance_rescale=0.7, sqrt_ac_t=0.6, sqrt_1mac_t=0.8, a_prev=0.5, sigma_t=0.3, scale_t=0.7, prev_scale_t=0.72)
xp, p0 = ops.ddim_update(xs, vc, vu, nz, sc)
torch.save(dict(y=y.cpu(), xp=xp.cpu(), p0=p0.cpu()), sys.argv[1])
"""


def test_results_do_not_depend_on_the_sm_count(tmp_path):
    """The full-width forward and a DDIM update with guidance rescale, as this device runs them and with every launch grid sized for
    a 114-SM H100 (VC_SM_COUNT only shrinks grids)."""
    script = tmp_path / "sm.py"
    script.write_text(_SM_SCRIPT.format(root=ROOT))
    outs = []
    for sms in (None, "114"):
        env = dict(os.environ, VC_REPRODUCIBLE="1")
        env.pop("VC_SM_COUNT", None)
        if sms:
            env["VC_SM_COUNT"] = sms
        f = tmp_path / f"out_{sms}.pt"
        r = subprocess.run([sys.executable, str(script), str(f)], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
        print(r.stdout[-1000:], r.stderr[-2000:])
        assert r.returncode == 0
        outs.append(torch.load(f))
    for k in ("y", "xp", "p0"):
        print(f"{k}: max |diff| between SM counts {float((outs[0][k] - outs[1][k]).abs().max()):.3g}")
        assert torch.equal(outs[0][k], outs[1][k]), k


def test_reproducible_on_two_gpus():
    """tools/reproducible_check.py under torch.distributed.run: frame sharding (peer memory and NCCL) and the CFG split, two-way and
    three-way guidance, bit-identical to one GPU."""
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} CUDA devices")
    for peer in ("1", "0"):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
               "--master-port", "29541", os.path.join(ROOT, "tools", "reproducible_check.py")]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, VC_PEER_COMM=peer, VC_REPRODUCIBLE="1"))
        print(r.stdout[-3000:], r.stderr[-2000:])
        assert r.returncode == 0 and "REPRODUCIBLE_CHECK_OK" in r.stdout
