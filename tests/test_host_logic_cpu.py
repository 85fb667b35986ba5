"""Host logic of the drop-in classes on the CPU: the CUDA ops are replaced by the torch test double (tests/fake_ops.py)
and the whole UNetModel / AutoencoderKL / DDIMSampler wiring is checked against the reference-generated goldens and the
oracle.  This does not test the kernels (the -m gpu suite does); it tests packing, layouts, block order and loops."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import lvdm_oracle as O
from oracle import synth
from tests import fake_ops
from viewcrafter_b200.configs import UNET_PARAMS, VAE_DDCONFIG


@pytest.fixture
def cpu_ops(monkeypatch):
    fake_ops.install(monkeypatch)
    return fake_ops


def test_product_refuses_cpu_without_the_double():
    from viewcrafter_b200 import _lib
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64)).eval()
    with pytest.raises(_lib.VcError):
        m(torch.zeros(1, 8, 2, 8, 8), torch.tensor([1]), context=torch.zeros(1, 333, 1024))


@pytest.mark.parametrize("name", ["mc64_T4", "mc64_T16"])
def test_unet_wiring_matches_reference_golden(cpu_ops, golden_dir, name):
    from viewcrafter_b200.unet import UNetModel
    g = np.load(os.path.join(golden_dir, f"unet_{name}.npz"))
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    kw = dict(UNET_PARAMS); kw.update(json.loads(str(g["kwargs"])))
    m = UNetModel(**kw).eval()
    m.load_state_dict(synth.synth_state_dict(shapes, 3), strict=True)
    y = m(torch.from_numpy(g["x"]), torch.from_numpy(g["t"]), context=torch.from_numpy(g["ctx"]).float(), fs=torch.from_numpy(g["fs"]))
    err = (y - torch.from_numpy(g["y"])).abs()
    assert float(err.max()) < 0.02 and float(err.mean()) < 0.003, (float(err.max()), float(err.mean()))


def test_unet_batch2_wiring(cpu_ops):
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64)).eval()
    sd = synth.synth_state_dict(synth.module_shapes(m), 9)
    m.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(10)
    x, ctx, t = torch.randn(2, 8, 3, 8, 8, generator=g), torch.randn(2, 333, 1024, generator=g), torch.tensor([999, 19])
    with torch.no_grad():
        ref = O.unet_forward(sd, x, t, ctx, None, default_fs=10)
    err = (m(x, t, context=ctx) - ref).abs()
    assert float(err.max()) < 0.02, float(err.max())


def test_vae_decode_wiring_matches_reference_golden(cpu_ops, golden_dir):
    from viewcrafter_b200.autoencoder import AutoencoderKL
    g = np.load(os.path.join(golden_dir, "vae_ch32.npz"))
    vae = AutoencoderKL(dict(VAE_DDCONFIG, ch=32), None, 4).eval()
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    sd = {"decoder." + k: v for k, v in synth.synth_state_dict(shapes, seed=4).items()}
    sd.update({"post_quant_conv." + k: v for k, v in synth.synth_state_dict([("weight", (4, 4, 1, 1)), ("bias", (4,))], 4).items()})
    missing, unexpected = vae.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith(("encoder.", "quant_conv.")) for k in missing)
    y = vae.decode(torch.from_numpy(g["z"]))
    err = (y - torch.from_numpy(g["y"])).abs()
    assert y.shape == g["y"].shape and float(err.max()) < 0.03, float(err.max())


@pytest.mark.parametrize("batch_cfg", [False, True])
def test_sampler_and_wrapper_wiring_vs_oracle(cpu_ops, batch_cfg):
    from viewcrafter_b200.ddim import DDIMSampler
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=dict(VAE_DDCONFIG, ch=32), embed_dim=4), base_scale=0.7).eval()
    unet = model.model.diffusion_model
    sd = synth.synth_state_dict(synth.module_shapes(unet), seed=41)
    unet.load_state_dict(sd, strict=True)
    sdv = synth.synth_state_dict(synth.module_shapes(model.first_stage_model), seed=44)
    model.first_stage_model.load_state_dict(sdv, strict=True)
    g = torch.Generator().manual_seed(42)
    T, H, W, S = 3, 8, 8, 2
    shape = (1, 4, T, H, W)
    x_T, cc = torch.randn(shape, generator=g), torch.randn(shape, generator=g)
    ctx_c, ctx_u = torch.randn(1, 333, 1024, generator=g), torch.randn(1, 333, 1024, generator=g)
    fs = torch.tensor([10])
    c = {"c_crossattn": [ctx_c], "c_concat": [cc]}
    uc = {"c_crossattn": [ctx_u], "c_concat": [cc]}
    sampler = DDIMSampler(model, batch_cfg=batch_cfg)
    torch.manual_seed(43)
    out, inter = sampler.sample(S=S, batch_size=1, shape=shape[1:], conditioning=c, eta=1.0, verbose=False, x_T=x_T,
                                unconditional_guidance_scale=7.5, unconditional_conditioning=uc, fs=fs,
                                timestep_spacing="uniform_trailing", guidance_rescale=0.7)
    torch.manual_seed(43)
    noises = [torch.randn(shape) for _ in range(S)]
    sched = O.model_schedule(base_scale=0.7)

    def model_fn(x, t, cond):
        with torch.no_grad():
            return O.unet_forward(sd, torch.cat([x, cc], 1), t, cond, fs)

    ref, _ = O.ddim_sample(model_fn, sched, shape, S, ctx_c, ctx_u, x_T, noises)
    err = (out - ref).abs()
    assert float(err.max()) < 0.15 and float(err.mean()) < 0.02, (float(err.max()), float(err.mean()))   # CFG 7.5 amplifies the fp16 U-Net error ~16x
    img = model.decode_first_stage(out)
    with torch.no_grad():
        ref_img = O.decode_first_stage(sdv, ref)
    assert img.shape == (1, 3, T, 8 * H, 8 * W)
    assert float((img - ref_img).abs().mean()) < 0.03 * max(1.0, float(ref_img.std()))


def test_latent_diffusion_builds_inside_cuda_device_context_guard():
    """model_buffers must not depend on torch's default device (bench builds the model under torch.device('cuda'))."""
    from viewcrafter_b200 import schedule
    with torch.device("meta"):
        b = schedule.model_buffers(base_scale=0.3)
    assert b["alphas_cumprod"].device.type == "cpu" and b["alphas_cumprod"].shape[0] == 1000


def test_shared_cfg_prefix_and_kv_cache(cpu_ops):
    """SURVEY.md App. C.1/C.2: the context-free prefix computed once and the cached cross-attention K/V give the results of the
    plain B=2 forward; the K/V cache follows the context tensor (new tensor or in-place write -> recomputed)."""
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64)).eval()
    m.load_state_dict(synth.synth_state_dict(synth.module_shapes(m), seed=51), strict=True)
    g = torch.Generator().manual_seed(52)
    x1 = torch.randn(1, 8, 3, 8, 8, generator=g)
    x = torch.cat([x1, x1], 0)
    t, fs = torch.tensor([499, 499]), torch.tensor([10, 10])
    ctx = torch.randn(2, 333, 1024, generator=g)
    plain = m(x, t, context=ctx, fs=fs)
    shared = m(x, t, context=ctx, fs=fs, cfg_shared_prefix=True)
    # not bit-equal: the fp16 roundings of a B=1 and a B=2 GEMM differ (summation order), the same noise as B=2 vs B=1 runs
    d = (plain - shared).abs()
    assert float(d.max()) < 0.02 and float(d.mean()) < 3e-3, (float(d.max()), float(d.mean()))
    assert float((plain[0] - plain[1]).abs().mean()) > 5 * float(d.mean())      # the two branches do differ (different context)
    # K/V cache: same tensor object -> hit; in-place change or a new tensor -> recomputed
    n_cached = len(m._kv_cache)
    assert n_cached > 3 and m._kv_cache["ref"] is ctx
    ctx2 = ctx.clone()
    ctx2[1] = ctx[0]
    out2 = m(x, t, context=ctx2, fs=fs)
    assert m._kv_cache["ref"] is ctx2
    assert float((out2[0] - out2[1]).abs().max()) < 0.02              # identical branches now
    ctx2[1] = ctx[1]                                                  # in-place write bumps the version counter
    out3 = m(x, t, context=ctx2, fs=fs)
    assert float((out3 - plain).abs().max()) < 0.02


def test_vae_encode_host_logic_vs_reference_golden(cpu_ops, golden_dir):
    """AutoencoderKL.encode (Encoder + folded conv_out/quant_conv + DiagonalGaussianDistribution) on the CPU op double vs the
    moments / posterior sample produced by the unmodified reference (tests/golden/vae_enc_ch32.npz)."""
    from viewcrafter_b200.autoencoder import AutoencoderKL
    g = np.load(os.path.join(golden_dir, "vae_enc_ch32.npz"))
    vae = AutoencoderKL(dict(VAE_DDCONFIG, ch=32), None, 4).eval()
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    sd = {"encoder." + k: v for k, v in synth.synth_state_dict(shapes, seed=14).items()}
    sd.update({"quant_conv." + k: v for k, v in synth.synth_state_dict([("weight", (8, 8, 1, 1)), ("bias", (8,))], 14).items()})
    missing, unexpected = vae.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith(("decoder.", "post_quant_conv.")) for k in missing)
    post = vae.encode(torch.from_numpy(g["x"]))
    err = (post.parameters - torch.from_numpy(g["moments"])).abs()
    assert post.parameters.shape == g["moments"].shape and float(err.max()) < 0.03, float(err.max())
    z = post.sample(noise=torch.from_numpy(g["noise"]))
    assert float((z - torch.from_numpy(g["z"])).abs().max()) < 0.05
    assert torch.equal(post.mode(), post.mean) and post.logvar.min() >= -30.0 and post.logvar.max() <= 20.0


def test_vae_odd_token_count_attention(cpu_ops):
    """A 40x72 image gives a 5x9 = 45-token mid AttnBlock: 45 is not a multiple of 8, so the key axis (a GEMM reduction
    and a row pitch) is padded with zero keys masked to -inf before the softmax.  The op double asserts the kernel's
    16-byte-stride contract, so an unpadded call fails here the way it fails on the GPU."""
    from viewcrafter_b200.autoencoder import AutoencoderKL
    vae = AutoencoderKL(dict(VAE_DDCONFIG, ch=32), None, 4).eval()
    sd = synth.synth_state_dict(synth.module_shapes(vae), seed=51)
    vae.load_state_dict(sd, strict=True)
    x = torch.rand(1, 3, 40, 72, generator=torch.Generator().manual_seed(52)) * 2 - 1
    with torch.no_grad():
        ref = O.vae_encode_moments(sd, x)
        m = vae.encode(x).parameters
        assert m.shape == ref.shape == (1, 8, 5, 9)
        assert float((m - ref).abs().max()) < 0.03
        z = torch.randn(1, 4, 5, 9, generator=torch.Generator().manual_seed(53))
        y, yr = vae.decode(z), O.vae_decode(sd, z)
        assert y.shape == yr.shape == (1, 3, 40, 72) and float((y - yr).abs().max()) < 0.03 * max(1.0, float(yr.std()))


def test_encode_first_stage_perframe_rng_order(cpu_ops):
    """LatentDiffusion.encode_first_stage: per-frame encodes, each drawing its posterior noise from the CPU generator in frame
    order (ddpm3d.py:633-639, distributions.py:35-36), scaled by scale_factor; checked against the oracle fed the same draws."""
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=dict(VAE_DDCONFIG, ch=32), embed_dim=4)).eval()
    sdv = synth.synth_state_dict(synth.module_shapes(model.first_stage_model), seed=45)
    model.first_stage_model.load_state_dict(sdv, strict=True)
    g = torch.Generator().manual_seed(46)
    x = torch.rand(1, 3, 3, 16, 24, generator=g) * 2 - 1
    torch.manual_seed(47)
    z = model.encode_first_stage(x)
    torch.manual_seed(47)
    noises = [torch.randn(1, 4, 2, 3) for _ in range(3)]
    with torch.no_grad():
        ref = O.encode_first_stage(sdv, x, noises)
    assert z.shape == (1, 4, 3, 2, 3)
    assert float((z - ref).abs().max()) < 0.02, float((z - ref).abs().max())


def test_resampler_wiring_matches_reference_golden(cpu_ops, golden_dir):
    """viewcrafter_b200.Resampler (image_proj_model, SURVEY.md 8f rank f3) on the CPU op double vs the output of the unmodified
    reference Resampler: same kwargs, same state-dict keys (strict load), same token order; B=2, 33 + 16 ragged keys."""
    from viewcrafter_b200.resampler import Resampler
    g = np.load(os.path.join(golden_dir, "resampler_d256.npz"))
    kw = json.loads(str(g["kwargs"]))
    m = Resampler(**kw).eval()
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == shapes          # names, shapes AND order of the reference
    m.load_state_dict(synth.synth_state_dict(shapes, seed=17), strict=True)
    y = m(torch.from_numpy(g["x"]))
    err = (y - torch.from_numpy(g["y"])).abs()
    assert y.shape == g["y"].shape and y.dtype == torch.float32
    assert float(err.max()) < 0.03 and float(err.mean()) < 0.004, (float(err.max()), float(err.mean()))
    with pytest.raises(NotImplementedError):
        Resampler(dim_head=32)


@pytest.mark.parametrize("tag,S,cfg_img", [("S5", 5, 2.5), ("S8", 8, None)])
def test_multicond_sampler_matches_reference_golden(cpu_ops, golden_dir, tag, S, cfg_img):
    """viewcrafter_b200.ddim_multiplecond.DDIMSampler (three apply_model calls, un-fixed scale_arr_prev[0]) driving the toy
    denoiser through the reference-shaped model interface vs the output of the unmodified reference sampler."""
    from viewcrafter_b200.ddim_multiplecond import DDIMSampler
    from viewcrafter_b200.diffusion import LatentDiffusion
    g = np.load(os.path.join(golden_dir, "ddim_multicond_small.npz"))
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.3).eval()
    calls = []

    def toy(x, t, c, **kw):
        calls.append(sorted(kw))
        return torch.tanh(0.7 * x * c["k"] + 0.05 * torch.sin(t.float())[:, None, None, None, None]) + 0.1 * c["b"]

    model.apply_model = toy
    noises = iter(torch.from_numpy(g[f"{tag}_noises"]))
    cond = {"k": torch.tensor([1.3]), "b": torch.from_numpy(g[f"{tag}_cond_b"])}
    unc = {"k": torch.tensor([0.4]), "b": torch.from_numpy(g[f"{tag}_uncond_b"])}
    unc_img = {"k": torch.tensor([0.9]), "b": torch.from_numpy(g[f"{tag}_uncond_img_b"])}
    import viewcrafter_b200.ddim_multiplecond as mod
    real_randn = torch.randn
    try:
        mod.torch.randn = lambda shape, device=None: next(noises)                       # inject the recorded per-step draws
        smp = DDIMSampler(model)
        out, inter = smp.sample(S=S, batch_size=1, shape=(4, 3, 4, 6), conditioning=cond, eta=1.0, verbose=False,
                                x_T=torch.from_numpy(g[f"{tag}_x_T"]), unconditional_guidance_scale=7.5,
                                unconditional_conditioning=unc, timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                                cfg_img=cfg_img, unconditional_conditioning_img_nonetext=unc_img)
    finally:
        mod.torch.randn = real_randn
    assert np.array_equal(smp.ddim_scale_arr_prev.numpy(), g[f"{tag}_scale_prev"])
    assert len(calls) == 3 * S and len(inter["x_inter"]) == int(g[f"{tag}_n_inter"])
    np.testing.assert_allclose(out.numpy(), g[f"{tag}_samples"], rtol=0, atol=5e-5)
    np.testing.assert_allclose(inter["pred_x0"][-1].numpy(), g[f"{tag}_pred_x0_last"], rtol=0, atol=5e-5)
    with pytest.raises(KeyError):                                                       # ddim_multiplecond.py:224 indexes kwargs
        smp.p_sample_ddim(torch.zeros(1, 4, 3, 4, 6), cond, torch.tensor([999]), index=S - 1)


@pytest.mark.parametrize("multi", [False, True])
def test_image_guided_synthesis_vs_oracle(cpu_ops, multi):
    """viewcrafter_b200.synthesis.image_guided_synthesis (utils/diffusion_utils.py:117-201): conditioning construction, hybrid
    concat of the per-frame encoded renders, CFG (2-way / 3-way), n_samples loop, decode and the [b, n, c, t, h, w] layout,
    with every RNG draw (posterior noise per frame, x_T, per-step noise, per sample) in the reference's order."""
    from viewcrafter_b200.diffusion import LatentDiffusion
    from viewcrafter_b200.synthesis import image_guided_synthesis
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), dict(ddconfig=dict(VAE_DDCONFIG, ch=32), embed_dim=4), base_scale=0.7).eval()
    sd = synth.synth_state_dict(synth.module_shapes(model.model.diffusion_model), seed=71)
    model.model.diffusion_model.load_state_dict(sd, strict=True)
    sdv = synth.synth_state_dict(synth.module_shapes(model.first_stage_model), seed=72)
    model.first_stage_model.load_state_dict(sdv, strict=True)
    g = torch.Generator().manual_seed(73)
    W_img, txt, txt_empty = torch.randn(3 * 4 * 4, 256 * 8, generator=g) * 0.1, torch.randn(1, 77, 1024, generator=g), torch.randn(1, 77, 1024, generator=g)
    model.embedder = lambda img: torch.nn.functional.adaptive_avg_pool2d(img, 4).reshape(img.shape[0], 1, -1)            # [b, 1, 48]
    model.image_proj_model = lambda e: (e @ W_img).reshape(e.shape[0], 256, 8).repeat(1, 1, 128)                           # [b, 256, 1024]
    model.get_learned_conditioning = lambda prompts: torch.cat([txt_empty if p == "" else txt for p in prompts], 0)
    model.uncond_type = "empty_seq"
    T, H, W, S, n_samples = 2, 8, 8, 2, 2
    videos = torch.rand(1, 3, T, 8 * H, 8 * W, generator=g) * 2 - 1
    shape = (1, 4, T, H, W)
    torch.manual_seed(74)
    out = image_guided_synthesis(model, ["a photo"], videos, list(shape), n_samples=n_samples, ddim_steps=S, ddim_eta=1.0,
                                 unconditional_guidance_scale=7.5, cfg_img=(2.0 if multi else None), fs=10, text_input=True,
                                 multiple_cond_cfg=multi, timestep_spacing="uniform_trailing", guidance_rescale=0.7, condition_index=[0])
    assert out.shape == (1, n_samples, 3, T, 8 * H, 8 * W)
    # replay the draws in the reference's order and rebuild the expected result with the oracle
    torch.manual_seed(74)
    enc_noise = [torch.randn(1, 4, H, W) for _ in range(T)]
    img = videos[:, :, 0]
    ctx = lambda t, im: torch.cat([t, model.image_proj_model(model.embedder(im))], 1)
    ctx_c, ctx_u, ctx_i = ctx(txt, img), ctx(txt_empty, torch.zeros_like(img)), ctx(txt_empty, img)
    fs = torch.tensor([10])
    with torch.no_grad():
        cc = O.encode_first_stage(sdv, videos, enc_noise)
    sched = O.model_schedule(base_scale=0.7)

    def model_fn(x, t, cond):
        with torch.no_grad():
            return O.unet_forward(sd, torch.cat([x, cc], 1), t, cond, fs)

    for k in range(n_samples):
        x_T = torch.randn(shape)
        noises = [torch.randn(shape) for _ in range(S)]
        extra = dict(fixed_prev_scale=False, uncond_img=ctx_i, cfg_img=2.0) if multi else {}
        ref, _ = O.ddim_sample(model_fn, sched, shape, S, ctx_c, ctx_u, x_T, noises, **extra)
        with torch.no_grad():
            ref_img = O.decode_first_stage(sdv, ref)
        err = (out[:, k] - ref_img).abs()
        assert float(err.mean()) < 0.03 * max(1.0, float(ref_img.std())), (k, float(err.mean()), float(ref_img.std()))


def test_posterior_class_subclasses_a_loaded_reference_class(monkeypatch):
    """AutoencoderKL.encode must return an instance of the reference's DiagonalGaussianDistribution whenever lvdm.distributions
    is loaded (ddpm3d.py:611-618 type-checks it); checked here with a stand-in module so that it also runs without /root/reference."""
    import sys
    import types
    from viewcrafter_b200 import distributions as D
    ref_mod = types.ModuleType("lvdm.distributions")

    class RefDGD(object):
        pass

    ref_mod.DiagonalGaussianDistribution = RefDGD
    monkeypatch.setitem(sys.modules, "lvdm.distributions", ref_mod)
    cls = D.posterior_class()
    post = cls(torch.zeros(1, 8, 2, 2))
    assert isinstance(post, RefDGD) and isinstance(post, D.DiagonalGaussianDistribution)
    assert D.posterior_class() is cls                                                   # cached per reference class
    assert post.sample(noise=torch.ones(1, 4, 2, 2)).shape == (1, 4, 2, 2)
    monkeypatch.delitem(sys.modules, "lvdm.distributions")
    assert D.posterior_class() is D.DiagonalGaussianDistribution


def test_upsample_conv_parity_decomposition_equals_interpolate_then_conv():
    """pack_upconv3x3: Upsample(nearest x2) + conv3x3 as four 2x2 sub-convolutions with pre-summed taps (openaimodel3d.py:80-106)."""
    import torch.nn.functional as F
    from tests import fake_ops
    g = torch.Generator().manual_seed(77)
    N, H, W, Ci, Co = 2, 5, 6, 8, 32
    x = torch.randn(N, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, 3, 3, generator=g) * 0.2
    b = torch.randn(Co, generator=g)
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, b, padding=1)
    rows = x.permute(0, 2, 3, 1).reshape(-1, Ci).half()
    y = fake_ops.upconv3x3(rows, N, H, W, fake_ops.pack_upconv3x3(w), bias=b)
    y = y.float().reshape(N, 2 * H, 2 * W, Co).permute(0, 3, 1, 2)
    ref16 = F.conv2d(F.interpolate(x.half().float(), scale_factor=2, mode="nearest"), w, b, padding=1)
    assert float((y - ref16).abs().max()) < 2e-2, float((y - ref16).abs().max())
    assert float((y - ref).abs().max()) < 3e-2


def test_groupnorm_partial_sum_geometry_of_every_producer_consumer_pair():
    """ops.GnPart.geom: which 32-row blocks of a producer's gn_part records make up sample s of the consuming GroupNorm
    (base = (s // samples_per_z) * rb_per_z + (s % samples_per_z) * rb_per_sample), or None when samples do not fall on block boundaries."""
    from viewcrafter_b200 import ops
    part = torch.zeros(8)

    def gp(X, Y, Z, bx, by, N=320):
        tx, ty = -(-X // bx), -(-Y // by)
        return ops.GnPart(part, N // 32, 10, tx * ty * 4, X * Y, Z, linear=(by == 1 and bx == 128 and (Y == 1 or X % 128 == 0)))

    def tup(g):
        return None if g is None else (g.rb_per_z, g.samples_per_z, g.rb_per_sample)

    T, B = 25, 2
    # 3x3 conv at 72x128 (one 128-pixel tile per image row): per-frame GroupNorm and the 5-D GroupNorm of the TemporalConvBlock
    c0 = gp(128, 72, B * T, 128, 1)
    assert tup(c0.geom(B * T, 72 * 128)) == (288, 1, 288)
    assert tup(c0.geom(B, T * 72 * 128)) == (T * 288, 1, T * 288)
    assert c0.geom(B * T + 1, 72 * 128) is None                                   # row count mismatch
    # 3x3 conv at 18x32 (tiles of 4 image rows, the fifth tile of a frame half empty): blocks are per frame, padding blocks hold zeros
    c2 = gp(32, 18, B * T, 32, 4)
    assert tup(c2.geom(B * T, 576)) == (20, 1, 20) and tup(c2.geom(B, T * 576)) == (T * 20, 1, T * 20)
    # temporal conv (X = T*HW rows per batch element, Z = B): 5-D consumer = one slab; per-frame consumer needs HW % 32 == 0
    t2 = gp(T * 576, 1, B, 128, 1)
    rbz = -(-T * 576 // 128) * 4
    assert tup(t2.geom(B, T * 576)) == (rbz, 1, rbz)
    assert tup(t2.geom(B * T, 576)) == (rbz, T, 18)
    t3 = gp(T * 144, 1, B, 128, 1)
    assert t3.geom(B * T, 144) is None and t3.geom(B, T * 144) is not None        # 144 rows per frame are not whole 32-row blocks
    # plain linear over all rows (one slab): frames and batch elements are runs of 32-row blocks when their row counts divide by 32
    l0 = gp(B * T * 2304, 1, 1, 128, 1)
    assert tup(l0.geom(B * T, 2304)) == (B * T * 2304 // 128 * 4, B * T, 72)
    assert tup(l0.geom(B, T * 2304)) == (B * T * 2304 // 128 * 4, B, T * 72)
    l3 = gp(B * T * 144, 1, 1, 128, 1)
    assert l3.geom(B * T, 144) is None and l3.geom(B, T * 144) is None            # 3600 rows per batch element: 112.5 blocks
    assert l3.geom(1, B * T * 144) is not None


def _toy_model(base):
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=base).eval()
    model.apply_model = lambda x, t, c, **kw: torch.tanh(0.7 * x * c["k"] + 0.05 * torch.sin(t.float())[:, None, None, None, None]) + 0.1 * c["b"]
    return model


def _with_recorded_noise(g, tag, fn):
    """Run fn() with torch.randn (the sampler's per-step draw) replaced by the recorded tensors of the reference run."""
    import viewcrafter_b200.ddim as mod
    noises = iter(torch.from_numpy(g[f"{tag}_noises"]))
    real = torch.randn
    try:
        mod.torch.randn = lambda shape, device=None: next(noises)
        return fn()
    finally:
        mod.torch.randn = real


@pytest.mark.parametrize("tag", ["mask", "maskclean", "subset", "dropout", "temp", "prec16", "batch2"])
def test_sampler_options_match_the_unmodified_reference_sampler(cpu_ops, golden_dir, tag):
    """The switches of DDIMSampler.sample / ddim_sampling beyond the ViewCrafter defaults -- mask / x0 blending (q_sample draw, clean_cond),
    a `timesteps` subset, noise_dropout (global-RNG dropout after the step draw), temperature, precision=16 (x_T rounded to fp16), batch 2
    with guidance rescale (per-sample statistics) -- against outputs of the unmodified reference sampler on the toy denoiser
    (tests/golden/ddim_options.npz, oracle/make_golden.py: gen_ddim_options)."""
    from viewcrafter_b200.ddim import DDIMSampler
    g = np.load(os.path.join(golden_dir, "ddim_options.npz"))
    model = _toy_model(0.5)
    x_T = torch.from_numpy(g[f"{tag}_x_T"])
    cond = {"k": torch.tensor([1.3]), "b": torch.from_numpy(g[f"{tag}_cond_b"])}
    unc = {"k": torch.tensor([0.4]), "b": torch.from_numpy(g[f"{tag}_uncond_b"])}
    smp = DDIMSampler(model)
    common = dict(batch_size=x_T.shape[0], shape=tuple(x_T.shape[1:]), eta=1.0, verbose=False, unconditional_guidance_scale=7.5,
                  timestep_spacing="uniform_trailing", guidance_rescale=0.7, conditioning=cond, x_T=x_T, unconditional_conditioning=unc)

    def run():
        if tag in ("mask", "maskclean"):
            torch.manual_seed(123)
            extra = dict(clean_cond=True) if tag == "maskclean" else {}
            return smp.sample(S=6, mask=torch.from_numpy(g[f"{tag}_mask"]), x0=torch.from_numpy(g[f"{tag}_x0"]), **extra, **common)
        if tag == "subset":
            smp.make_schedule(ddim_num_steps=10, ddim_discretize="uniform_trailing", ddim_eta=1.0, verbose=False)
            return smp.ddim_sampling(cond, tuple(x_T.shape), x_T=x_T, timesteps=6, unconditional_guidance_scale=7.5,
                                     unconditional_conditioning=unc, verbose=False, guidance_rescale=0.7)
        if tag == "dropout":
            torch.manual_seed(321)
            return smp.sample(S=5, noise_dropout=0.25, **common)
        if tag == "temp":
            return smp.sample(S=5, temperature=0.6, **common)
        if tag == "prec16":
            return smp.sample(S=5, precision=16, **common)
        return smp.sample(S=5, **common)

    out, inter = _with_recorded_noise(g, tag, run)
    assert len(inter["x_inter"]) == int(g[f"{tag}_n_inter"])
    np.testing.assert_allclose(out.float().numpy(), g[f"{tag}_samples"], rtol=0, atol=5e-5)
    np.testing.assert_allclose(inter["pred_x0"][-1].float().numpy(), g[f"{tag}_pred_x0_last"], rtol=0, atol=5e-5)
    if tag == "prec16":
        assert str(inter["x_inter"][0].dtype) == str(g["prec16_first_inter_dtype"]) == "torch.float16" and out.dtype == torch.float32


def test_sampler_decode_and_stochastic_encode_match_the_reference(cpu_ops, golden_dir):
    """DDIMSampler.decode (the last t_start steps from a given latent) and stochastic_encode (q(x_t | x_0) from the DDIM tables), ddim.py:288-325."""
    from viewcrafter_b200.ddim import DDIMSampler
    g = np.load(os.path.join(golden_dir, "ddim_options.npz"))
    model = _toy_model(0.5)
    x = torch.from_numpy(g["decode_x_T"])
    cond = {"k": torch.tensor([1.3]), "b": torch.from_numpy(g["decode_cond_b"])}
    unc = {"k": torch.tensor([0.4]), "b": torch.from_numpy(g["decode_uncond_b"])}
    smp = DDIMSampler(model)
    smp.make_schedule(ddim_num_steps=8, ddim_discretize="uniform_trailing", ddim_eta=1.0, verbose=False)
    seen = []
    dec = _with_recorded_noise(g, "decode", lambda: smp.decode(x, cond, 5, unconditional_guidance_scale=7.5, unconditional_conditioning=unc,
                                                                callback=seen.append))
    assert seen == [0, 1, 2, 3, 4]
    np.testing.assert_allclose(dec.numpy(), g["decode_samples"], rtol=0, atol=5e-5)
    enc = smp.stochastic_encode(torch.from_numpy(g["stoch_x0"]), torch.tensor([3]), noise=torch.from_numpy(g["stoch_noise"]))
    np.testing.assert_allclose(enc.numpy(), g["stoch_out"], rtol=0, atol=1e-6)


def test_sampler_options_the_reference_cannot_run_either_raise(cpu_ops):
    from viewcrafter_b200.ddim import DDIMSampler
    smp = DDIMSampler(_toy_model(0.5))
    smp.make_schedule(4, "uniform_trailing", 1.0, verbose=False)
    x, c, t = torch.zeros(1, 4, 3, 4, 6), {"k": torch.tensor([1.0]), "b": torch.zeros(1, 4, 3, 4, 6)}, torch.tensor([999])
    with pytest.raises(NotImplementedError):
        smp.ddim_sampling(c, x.shape, ddim_use_original_steps=True)                    # ddim.py:248 reads an attribute that is never set
    with pytest.raises(NotImplementedError):
        smp.p_sample_ddim(x, c, t, index=3, quantize_denoised=True)                    # needs a VQ first stage
    with pytest.raises(AssertionError):
        smp.p_sample_ddim(x, c, t, index=3, score_corrector=object())                  # ddim.py:240 asserts the eps parameterisation
