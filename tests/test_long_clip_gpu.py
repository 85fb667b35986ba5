"""Clips of 33..128 frames on the GPU: the long-clip temporal-attention kernel, the U-Net and the samplers at T > 32.

Kernel: `temporal_attn` at 33 <= T <= 128 against float64 through the bound of `tests/attention_ref.py` (worst |out - ref| / bound <= 1,
as in `tests/test_attention_numerics_gpu.py`), on the rungs that exist for T keys, site counts that leave CTAs without work, and the
level-0 call where the grid strides.  The GEGLU linear of the level-0 transformer at 576x1024, B = 3 and T = 61 writes more than 2^31
elements.  U-Net: the reference golden at T = 48 and the fp32 oracle at T = 40 / 49 within the bounds of `tests/test_unet_gpu.py`; graph
replay at T = 49.  Samplers: `image_guided_synthesis` on a 49-frame clip against the oracle pipeline, and DPM-Solver++(2M) against DDIM.
Multi-GPU: `tools/long_clip_check.py` on 2 and 4 ranks (skipped with fewer devices).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import attention_ref as ar
from tests.test_attention_numerics_gpu import temporal_case

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_ERR, MEAN_ERR = 0.02, 0.003          # the U-Net forward bounds of test_unet_gpu.py
HW0, HEADS0 = 72 * 128, 5                # level 0 at 576x1024


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


def _check(r, what):
    print(f"{what}: worst |out - ref| / bound = {r:.3g}")
    assert r <= 1.0, f"{what}: |out - ref| / bound = {r:.4g}"


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("rung", ["centred", "peaked16"])
@pytest.mark.parametrize("T", [33, 40, 48, 49, 63, 64, 65, 96, 127, 128])
def test_long_temporal_attn_T(ops, T, rung):
    _check(temporal_case(ops, rung, 1, T, 33, 2, seed=T), f"T={T} {rung}")


@pytest.mark.parametrize("T", [49, 128])
def test_long_temporal_attn_rungs(ops, T):
    for rung in ar.rungs_for(T):
        _check(temporal_case(ops, rung, 2, T, 144, 5, seed=41), f"T={T} {rung}")


@pytest.mark.parametrize("T", [33, 80, 128])
@pytest.mark.parametrize("sites", [1, 7, 33])
def test_long_temporal_attn_partial_ctas(ops, T, sites):
    """3 heads: a CTA per pair with fewer 16-row query tiles than warps (T = 33), or more (T = 80, 128), and fewer pairs than CTAs."""
    for rung in ("centred", "shift-30", "late-max@last"):
        _check(temporal_case(ops, rung, 1, T, sites, 3, seed=sites), f"T={T} sites={sites} {rung}")


@pytest.mark.parametrize("rung", ["centred", "peaked16", "shift-30", "v-offset"])
def test_long_temporal_attn_level0(ops, rung):
    """9216 sites x 5 heads per batch element at T = 49: far more pairs than resident CTAs, so every CTA strides."""
    _check(temporal_case(ops, rung, 2, 49, HW0, HEADS0, seed=43), f"level0 T=49 {rung}")


@pytest.mark.parametrize("T", [0, 129])
def test_long_temporal_attn_rejects_T(ops, T):
    q = torch.zeros((64, 3 * 64), device="cuda", dtype=torch.float16)
    out = torch.full((T * 2, 64), 7.0, device="cuda", dtype=torch.float16) if T else torch.zeros((0, 64), device="cuda",
                                                                                                 dtype=torch.float16)
    with pytest.raises(ops.VcError, match=r"T=%d unsupported \(1\.\.128\)" % T):
        ops.temporal_attn(q[:, :64], q[:, 64:128], q[:, 128:], T, 2, 1, out=out)
    torch.cuda.synchronize()
    assert T == 0 or bool((out == 7.0).all())           # nothing was launched


def test_geglu_past_2e31_elements(ops):
    """Level-0 GEGLU of a B = 3, T = 61 clip at 576x1024: 3 * 61 * 9216 rows x 1280 outputs = 2.16e9 elements.  The rows whose
    element offsets pass 2^31 are checked against torch on the same fp16 operands."""
    rows, C, inner = 3 * 61 * HW0, 320, 1280
    assert rows * inner > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(7)
    x = (torch.randn(rows, C, generator=g, device="cuda") * 0.5).half()
    w = torch.randn(2 * inner, C, generator=g, device="cuda") * C ** -0.5
    b = torch.randn(2 * inner, generator=g, device="cuda") * 0.1
    wp, bp = ops.pack_geglu(w, b)
    y = ops.linear(x, wp, bias=bp, geglu=True)
    assert y.shape == (rows, inner)
    first = 2 ** 31 // inner
    sel = torch.cat([torch.arange(0, 64), torch.arange(first - 64, first + 64), torch.arange(rows - 64, rows)]).cuda()
    h = x[sel].float() @ w.half().float().t() + b
    ref = h[:, :inner] * torch.nn.functional.gelu(h[:, inner:])
    err = float((y[sel].float() - ref).abs().max())
    print(f"GEGLU {rows} x {inner}: max |err| on the rows around 2^31 elements {err:.3g}")
    assert err < 2e-2 * max(1.0, float(ref.abs().max()))
    del x, y


# ------------------------------------------------------------------------------------------------ U-Net
def _unet(seed, **over):
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64, **over))
    sd = synth.synth_state_dict(synth.module_shapes(m), seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


def test_unet_T48_matches_reference_golden(golden_dir, ops):
    from oracle import synth
    from tests.test_unet_gpu import _build
    g = np.load(os.path.join(golden_dir, "unet_mc64_T48.npz"))
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    m, _ = _build(json.loads(str(g["kwargs"])), shapes, seed=3)
    assert g["x"].shape[2] == 48 and g["ctx"].shape[1] != 77 + 16 * 48       # shared image tokens
    y = m(torch.from_numpy(g["x"]).cuda(), torch.from_numpy(g["t"]).cuda(), context=torch.from_numpy(g["ctx"]).float().cuda(),
          fs=torch.from_numpy(g["fs"]).cuda())
    err = (y.cpu() - torch.from_numpy(g["y"])).abs()
    print(f"mc64_T48: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g}")
    assert y.shape == g["y"].shape and torch.isfinite(y).all()
    assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR


def test_unet_T40_per_frame_tokens_batch2_vs_oracle(ops):
    """B = 2 at T = 40 with a per-frame image context (L = 77 + 16 T)."""
    from oracle import lvdm_oracle as O
    m, sd = _unet(9)
    g = torch.Generator().manual_seed(10)
    T = 40
    x, ctx = torch.randn(2, 8, T, 8, 8, generator=g), torch.randn(2, 77 + 16 * T, 1024, generator=g)
    t, fs = torch.tensor([999, 19]), torch.tensor([10, 10])
    with torch.no_grad():
        ref = O.unet_forward(sd, x, t, ctx, fs)
    y = m(x.cuda(), t.cuda(), context=ctx.cuda(), fs=fs.cuda())
    err = (y.cpu() - ref).abs()
    print(f"T=40 B=2 per-frame tokens: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g}")
    assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR


def test_unet_T49_shared_prefix_vs_oracle_and_graph_replay(ops):
    """The shared-CFG-prefix B = 2 forward at T = 49 against the oracle; then graph replay equal to it bit for bit, B = 2 and B = 3."""
    from oracle import lvdm_oracle as O
    m, sd = _unet(11)
    g = torch.Generator().manual_seed(12)
    T = 49
    x1 = torch.randn(1, 8, T, 8, 8, generator=g)
    ctx = torch.randn(3, 333, 1024, generator=g)
    with torch.no_grad():
        ref = O.unet_forward(sd, torch.cat([x1, x1], 0), torch.tensor([499, 499]), ctx[:2], torch.tensor([10, 10]))
    for B in (2, 3):
        x, cc = torch.cat([x1] * B, 0).cuda(), ctx[:B].cuda()
        t, fs = torch.full((B,), 499).cuda(), torch.full((B,), 10).cuda()
        m.enable_cuda_graph(False)
        eager = m(x, t, context=cc, fs=fs, cfg_shared_prefix=True)
        if B == 2:
            err = (eager.cpu() - ref).abs()
            print(f"T=49 shared prefix: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g}")
            assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR
        m.enable_cuda_graph()
        for _ in range(3):                                          # eager, capture, replay
            y = m(x, t, context=cc, fs=fs, cfg_shared_prefix=True)
            assert torch.equal(y, eager), (B, float((y - eager).abs().max()))
        assert any(e["graph"] is not None for e in m._graphs.values())
    m.enable_cuda_graph(False)


# ------------------------------------------------------------------------------------------------ samplers
@pytest.mark.parametrize("multi", [False, True])
def test_image_guided_synthesis_49_frames_vs_oracle(multi):
    """image_guided_synthesis on a 49-frame clip (VAE encode, batched CFG DDIM with graph replay, VAE decode), two-way and three-way,
    3 steps, against the oracle pipeline fed the same draws, in the manner of test_pipeline_gpu.py."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import lvdm_oracle as O
    from oracle import synth
    from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG
    from viewcrafter_b200.diffusion import LatentDiffusion
    from viewcrafter_b200.synthesis import image_guided_synthesis
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=dict(VAE_DDCONFIG, ch=32), embed_dim=4), base_scale=0.7).eval()
    sd = synth.synth_state_dict(synth.module_shapes(model.model.diffusion_model), seed=71)
    model.model.diffusion_model.load_state_dict(sd, strict=True)
    sdv = synth.synth_state_dict(synth.module_shapes(model.first_stage_model), seed=72)
    model.first_stage_model.load_state_dict(sdv, strict=True)
    model = model.cuda()
    g = torch.Generator().manual_seed(73)
    W_img, txt, txt_empty = torch.randn(3 * 4 * 4, 256 * 8, generator=g) * 0.1, torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)
    W_d, txt_d, txt_empty_d = W_img.cuda(), txt.cuda(), txt_empty.cuda()
    model.embedder = lambda img: torch.nn.functional.adaptive_avg_pool2d(img, 4).reshape(img.shape[0], 1, -1)
    model.image_proj_model = lambda e: (e @ (W_d if e.is_cuda else W_img)).reshape(e.shape[0], 256, 8).repeat(1, 1, 128)
    model.get_learned_conditioning = lambda prompts: torch.cat([txt_empty_d if p == "" else txt_d for p in prompts], 0)
    model.uncond_type = "empty_seq"
    T, H, W, S, n_samples = 49, 8, 8, 3, 1
    videos = torch.rand(1, 3, T, 8 * H, 8 * W, generator=g) * 2 - 1
    shape = (1, 4, T, H, W)
    torch.manual_seed(74)
    out = image_guided_synthesis(model, ["a photo"], videos.cuda(), list(shape), n_samples=n_samples, ddim_steps=S, ddim_eta=1.0,
                                 unconditional_guidance_scale=7.5, cfg_img=(2.0 if multi else None), fs=10, text_input=True,
                                 multiple_cond_cfg=multi, timestep_spacing="uniform_trailing", guidance_rescale=0.7, condition_index=[0])
    assert out.shape == (1, n_samples, 3, T, 8 * H, 8 * W) and out.is_cuda and bool(torch.isfinite(out).all())
    torch.manual_seed(74)
    enc_noise = [torch.randn(1, 4, H, W) for _ in range(T)]
    img = videos[:, :, 0]
    ctx = lambda t, im: torch.cat([t, model.image_proj_model(model.embedder(im))], 1)
    ctx_c, ctx_u, ctx_i = ctx(txt, img), ctx(txt_empty, torch.zeros_like(img)), ctx(txt_empty, img)
    fs = torch.tensor([10])
    torch.set_num_threads(max(1, min(os.cpu_count() or 1, 16)))
    with torch.no_grad():
        cc = O.encode_first_stage(sdv, videos, enc_noise)
    sched = O.model_schedule(base_scale=0.7)

    def model_fn(x, t, cond):
        with torch.no_grad():
            return O.unet_forward(sd, torch.cat([x, cc], 1), t, cond, fs)

    x_T = torch.randn(shape, device="cuda").cpu()
    noises = [torch.randn(shape, device="cuda").cpu() for _ in range(S)]
    extra = dict(fixed_prev_scale=False, uncond_img=ctx_i, cfg_img=2.0) if multi else {}
    ref, _ = O.ddim_sample(model_fn, sched, shape, S, ctx_c, ctx_u, x_T, noises, **extra)
    with torch.no_grad():
        ref_img = O.decode_first_stage(sdv, ref)
    err = (out[:, 0].cpu() - ref_img).abs()
    print(f"synthesis T=49 multi={multi}: mean err {float(err.mean()):.4g} max {float(err.max()):.4g} ref std {float(ref_img.std()):.3g}")
    assert float(err.mean()) < 0.05 * max(1.0, float(ref_img.std()))


@pytest.mark.parametrize("three_way", [False, True])
def test_dpmpp_2m_two_steps_equal_ddim_at_49_frames(three_way):
    """Both steps of a 2-step DPM-Solver++(2M) run are first order: bit-identical to DDIM with the same seed."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from tests.test_dpm_solver_gpu import _classes, _ld_model
    model = _ld_model()
    g = torch.Generator().manual_seed(42)
    shape = (1, 4, 49, 8, 8)
    x_T, cc = torch.randn(shape, generator=g).cuda(), torch.randn(shape, generator=g).cuda()
    c, uc, ui = ({"c_crossattn": [torch.randn(1, 333, 1024, generator=g).cuda()], "c_concat": [cc]} for _ in range(3))
    outs = []
    for cls in _classes(three_way):
        kw = dict(cfg_img=2.0, unconditional_conditioning_img_nonetext=ui) if three_way else {}
        torch.manual_seed(43)
        out, inter = cls(model, batch_cfg=True).sample(
            S=2, batch_size=1, shape=shape[1:], conditioning=c, eta=1.0, verbose=False, x_T=x_T, log_every_t=1,
            unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=torch.tensor([10]).cuda(),
            timestep_spacing="uniform_trailing", guidance_rescale=0.7, **kw)
        outs.append((out, inter["pred_x0"][-1]))
    (a, pa), (b, pb) = outs
    assert a.shape == shape and bool(torch.isfinite(a).all())
    assert torch.equal(a, b) and torch.equal(pa, pb)


# ------------------------------------------------------------------------------------------------ multi-GPU
@pytest.mark.parametrize("world,peer", [(2, "1"), (2, "0"), (4, "1"), (4, "0")])
def test_long_clip_multi_gpu(world, peer):
    """tools/long_clip_check.py: the frame-sharded T = 49 forward against one GPU, and reproducible mode on 1 / 2 / 4 GPUs."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} CUDA devices")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tools", "long_clip_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=850, env=dict(os.environ, VC_PEER_COMM=peer))
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0 and "LONG_CLIP_CHECK_OK" in r.stdout
