"""U-Net parity on the GPU: viewcrafter_b200.UNetModel (CUDA kernels via the C ABI) vs
  (a) golden outputs of the UNMODIFIED reference UNetModel (tests/golden/unet_*.npz, fp32 CPU), and
  (b) the CPU oracle on the same seeded inputs.

Tolerance (stated): activations are fp16 with fp32 accumulation, the reference runs the
same graph under torch.cuda.amp.autocast (fp16 GEMMs, fp32 norms).  For these synthetic weights the output has
std ~0.5-0.6; we require max|err| <= 0.02 and mean|err| <= 0.003 against the fp32 reference (measured: 0.007 / 0.0012), i.e. < 4% / 0.6% of
the output std -- the level autocast itself sits at for a ~150-GEMM-deep fp16 network.
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

UNET_KW = dict(in_channels=8, out_channels=4, model_channels=320, attention_resolutions=[4, 2, 1],
               num_res_blocks=2, channel_mult=[1, 2, 4, 4], dropout=0.1, num_head_channels=64,
               transformer_depth=1, context_dim=1024, use_linear=True, use_checkpoint=False,
               temporal_conv=True, temporal_attention=True, temporal_selfatt_only=True,
               use_relative_position=False, use_causal_attention=False, temporal_length=16,
               addition_attention=True, image_cross_attention=True, default_fs=10, fs_condition=True)

MAX_ERR, MEAN_ERR = 0.02, 0.003


def _build(over, shapes, seed):
    from oracle import synth
    from viewcrafter_b200.unet import UNetModel
    kw = dict(UNET_KW); kw.update(over)
    m = UNetModel(**kw)
    sd = synth.synth_state_dict(shapes, seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


@pytest.mark.parametrize("name", ["mc64_T4", "mc64_T16", "mc128_T3"])
def test_unet_matches_reference_golden(golden_dir, name):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    g = np.load(os.path.join(golden_dir, f"unet_{name}.npz"))
    shapes = [(n, tuple(s)) for n, s in json.loads(str(g["shapes"]))]
    m, _ = _build(json.loads(str(g["kwargs"])), shapes, seed=3)
    y = m(torch.from_numpy(g["x"]).cuda(), torch.from_numpy(g["t"]).cuda(), context=torch.from_numpy(g["ctx"]).float().cuda(),
          fs=torch.from_numpy(g["fs"]).cuda())
    err = (y.cpu() - torch.from_numpy(g["y"])).abs()
    print(f"{name}: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g} ref std {float(g['y'].std()):.3g}")
    assert y.shape == g["y"].shape and torch.isfinite(y).all()
    assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR


def test_unet_batch2_and_default_fs_vs_oracle():
    """B=2 (two independent latents/contexts) with fs=None (default_fs path) against the CPU oracle."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import lvdm_oracle as O
    from oracle import synth
    from viewcrafter_b200.unet import UNetModel
    kw = dict(UNET_KW); kw.update(model_channels=64)
    m = UNetModel(**kw)
    shapes = synth.module_shapes(m)
    m, sd = _build(dict(model_channels=64), shapes, seed=9)
    g = torch.Generator().manual_seed(10)
    x = torch.randn(2, 8, 5, 8, 8, generator=g)
    ctx = torch.randn(2, 333, 1024, generator=g)
    t = torch.tensor([999, 19])
    with torch.no_grad():
        ref = O.unet_forward(sd, x, t, ctx, None, default_fs=10)
    y = m(x.cuda(), t.cuda(), context=ctx.cuda())
    err = (y.cpu() - ref).abs()
    print(f"B=2: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g}")
    assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR


def test_shared_cfg_prefix_vs_oracle():
    """cond/uncond batch with the context-free prefix computed once (cfg_shared_prefix, SURVEY.md App. C.2) and the cached
    cross-attention K/V (App. C.1): same outputs as two independent oracle forwards, also on the second (cache-hit) call."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import lvdm_oracle as O
    from oracle import synth
    from viewcrafter_b200.unet import UNetModel
    kw = dict(UNET_KW); kw.update(model_channels=64)
    shapes = synth.module_shapes(UNetModel(**kw))
    m, sd = _build(dict(model_channels=64), shapes, seed=11)
    g = torch.Generator().manual_seed(12)
    x1 = torch.randn(1, 8, 5, 8, 8, generator=g)
    x = torch.cat([x1, x1], 0)
    ctx = torch.randn(2, 333, 1024, generator=g)
    t, fs = torch.tensor([499, 499]), torch.tensor([10, 10])
    with torch.no_grad():
        ref = O.unet_forward(sd, x, t, ctx, fs)
    xc, tc, cc, fc = x.cuda(), t.cuda(), ctx.cuda(), fs.cuda()
    for call in range(2):
        y = m(xc, tc, context=cc, fs=fc, cfg_shared_prefix=True)
        err = (y.cpu() - ref).abs()
        print(f"shared prefix call {call}: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g}")
        assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR
    assert torch.equal(m._kv_cache["ref"], cc) and len(m._kv_cache) > 3   # keyed on a private snapshot of the context


def test_unet_full_width_block_stack_vs_oracle():
    """Real channel widths (model_channels=320: 5/10/20 heads, N tiles of 160/256, K split 1280+640...) at a tiny
    spatial size so the fp32 CPU oracle finishes in seconds."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import lvdm_oracle as O
    from oracle import synth
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**UNET_KW)
    shapes = synth.module_shapes(m)
    del m
    m, sd = _build({}, shapes, seed=12)
    g = torch.Generator().manual_seed(13)
    x = torch.randn(1, 8, 3, 8, 16, generator=g)
    ctx = torch.randn(1, 333, 1024, generator=g)
    t, fs = torch.tensor([499]), torch.tensor([10])
    torch.set_num_threads(max(1, min(os.cpu_count() or 1, 16)))
    with torch.no_grad():
        ref = O.unet_forward(sd, x, t, ctx, fs)
    y = m(x.cuda(), t.cuda(), context=ctx.cuda(), fs=fs.cuda())
    err = (y.cpu() - ref).abs()
    print(f"mc320: max err {float(err.max()):.4g} mean err {float(err.mean()):.4g} ref std {float(ref.std()):.3g}")
    assert float(err.max()) <= MAX_ERR and float(err.mean()) <= MEAN_ERR


def test_cuda_graph_replay_is_bit_identical_to_eager():
    """enable_cuda_graph(): call 1 runs eagerly, call 2 captures, calls 3+ replay -- with different x / t each call; every result
    must equal the eager forward bit for bit (same kernels in the same order), also with the shared-CFG-prefix batch."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import synth
    from viewcrafter_b200.unet import UNetModel
    kw = dict(UNET_KW); kw.update(model_channels=64)
    shapes = synth.module_shapes(UNetModel(**kw))
    m, _ = _build(dict(model_channels=64), shapes, seed=31)
    g = torch.Generator().manual_seed(32)
    ctx = torch.randn(2, 333, 1024, generator=g).cuda()
    fs = torch.tensor([10, 10]).cuda()
    xs = [torch.randn(1, 8, 5, 8, 16, generator=g).cuda() for _ in range(4)]
    ts = [torch.tensor([t, t]).cuda() for t in (999, 979, 499, 19)]
    eager = [m(torch.cat([x, x], 0), t, context=ctx, fs=fs, cfg_shared_prefix=True) for x, t in zip(xs, ts)]
    m.enable_cuda_graph()
    for i, (x, t) in enumerate(zip(xs, ts)):
        y = m(torch.cat([x, x], 0), t, context=ctx, fs=fs, cfg_shared_prefix=True)
        assert torch.equal(y, eager[i]), (i, float((y - eager[i]).abs().max()))
    assert sum(e["graph"] is not None for e in m._graphs.values()) == 1
    ctx.add_(0.25)                                                      # in-place write to the context: the graph must not be reused
    y = m(torch.cat([xs[0], xs[0]], 0), ts[0], context=ctx, fs=fs, cfg_shared_prefix=True)
    m.enable_cuda_graph(False)
    ref = m(torch.cat([xs[0], xs[0]], 0), ts[0], context=ctx, fs=fs, cfg_shared_prefix=True)
    assert torch.equal(y, ref) and not torch.equal(y, eager[0])


def test_equal_context_rebuilt_every_call_hits_the_caches():
    """The reference's DiffusionWrapper concatenates c_crossattn anew on every call (ddpm3d.py:1442): a fresh tensor with the same
    content must reuse the K/V projections and the captured graph (content-keyed snapshot), and give the same output."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import synth
    from viewcrafter_b200.unet import UNetModel
    kw = dict(UNET_KW); kw.update(model_channels=64)
    shapes = synth.module_shapes(UNetModel(**kw))
    m, _ = _build(dict(model_channels=64), shapes, seed=33)
    g = torch.Generator().manual_seed(34)
    ctx = torch.randn(1, 333, 1024, generator=g).cuda()
    x = torch.randn(1, 8, 4, 8, 16, generator=g).cuda()
    t, fs = torch.tensor([499]).cuda(), torch.tensor([10]).cuda()
    ref = m(x, t, context=ctx, fs=fs)
    m.enable_cuda_graph()
    outs = [m(x, t, context=torch.cat([ctx[:, :77], ctx[:, 77:]], 1), fs=fs) for _ in range(4)]
    assert all(torch.equal(o, ref) for o in outs)
    assert len(m._canon) == 1 and len(m._kv_caches) == 1
    assert sum(e["graph"] is not None for e in m._graphs.values()) == 1
