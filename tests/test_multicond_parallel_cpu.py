"""Three-way classifier-free guidance (ddim_multiplecond.DDIMSampler) as one batched forward and on several ranks, on the CPU:
gloo process groups, CUDA ops replaced by the torch double (tests/fake_ops.py).  Checks that
  * the B=3 (cond, uncond, uncond_img) forward gives the step of the B=2 + B=1 forwards, and its stacked context is built once
    per clip (so the U-Net's K/V cache sees the same tensor every step);
  * a three-way step under shard_model -- 2-way CFG split (cond on one half of the ranks, uncond + uncond_img on the other) and
    pure frame sharding (the B=3 forward over all ranks) -- matches the single-process step."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import synth
from viewcrafter_b200.configs import UNET_PARAMS


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _problem(T=4):
    from viewcrafter_b200.diffusion import LatentDiffusion
    model = LatentDiffusion(dict(UNET_PARAMS, model_channels=64), None, base_scale=0.3).eval()
    unet = model.model.diffusion_model
    unet.load_state_dict(synth.synth_state_dict(synth.module_shapes(unet), 7), strict=True)
    g = torch.Generator().manual_seed(8)
    shape = (1, 4, T, 16, 16)
    x, cc = torch.randn(shape, generator=g), torch.randn(shape, generator=g)
    c = {"c_crossattn": [torch.randn(1, 333, 1024, generator=g)], "c_concat": [cc]}
    uc = {"c_crossattn": [torch.randn(1, 333, 1024, generator=g)], "c_concat": [cc]}
    ui = {"c_crossattn": [torch.randn(1, 333, 1024, generator=g)], "c_concat": [cc]}
    return model, x, c, uc, ui


def _step(sampler, x, c, uc, ui, index=2, t=599):
    sampler.make_schedule(5, "uniform_trailing", 1.0, verbose=False)
    torch.manual_seed(9)
    return sampler.p_sample_ddim(x, c, torch.full((1,), t, dtype=torch.long), index=index, unconditional_guidance_scale=7.5,
                                 unconditional_conditioning=uc, cfg_img=2.0, unconditional_conditioning_img_nonetext=ui,
                                 fs=torch.tensor([10]), guidance_rescale=0.7)


def _record_batches(model):
    """Wrap model.apply_model to record the batch size of every U-Net call."""
    seen, inner = [], model.apply_model

    def apply_model(x, t, cond, **kw):
        seen.append((x.shape[0], bool(kw.get("cfg_shared_prefix"))))
        return inner(x, t, cond, **kw)
    model.apply_model = apply_model
    return seen


def test_three_way_step_as_one_batch3_forward(monkeypatch):
    from tests import fake_ops
    from viewcrafter_b200.ddim_multiplecond import DDIMSampler
    fake_ops.install(monkeypatch)
    model, x, c, uc, ui = _problem()
    seen = _record_batches(model)

    class TwoPlusOne(DDIMSampler):                     # the path taken when the three conditionings do not stack
        def _can_stack(self, *conds):
            return len(conds) == 2 and super()._can_stack(*conds)

    ref = _step(TwoPlusOne(model, batch_cfg=True), x, c, uc, ui)
    assert seen == [(2, True), (1, False)]
    del seen[:]
    smp = DDIMSampler(model, batch_cfg=True)
    out = _step(smp, x, c, uc, ui)
    assert seen == [(3, True)]
    d = max(float((a - b).abs().max()) for a, b in zip(out, ref))
    print(f"B=3 step vs B=2 + B=1 step: max |diff| {d:.3g}")
    assert d < 0.15, d                                 # different GEMM batch sizes: fp16 rounding noise, amplified by CFG 7.5
    # the stacked conditioning is built once and reused by the next step: the U-Net's K/V cache keys on that one tensor
    unet = model.model.diffusion_model
    cat, kv0 = smp._cat_cache[2], unet._kv_cache
    assert kv0["ref"] is cat["c_crossattn"][0]
    _step(smp, out[0], c, uc, ui, index=1, t=399)
    assert smp._cat_cache[2] is cat and unet._kv_cache is kv0           # same stacked tensor -> the projections are reused
    # an in-place write to one branch's context is seen (version counter): the stack is rebuilt
    ui["c_crossattn"][0].add_(0.0)
    _step(smp, out[0], c, uc, ui, index=1, t=399)
    assert smp._cat_cache[2] is not cat
    # batch_cfg=False keeps the reference's three separate forwards
    del seen[:]
    _step(DDIMSampler(model, batch_cfg=False), x, c, uc, ui)
    assert seen == [(1, False)] * 3


def test_three_way_sampler_accepts_the_cfg_split(monkeypatch):
    """The three-way sampler used to raise NotImplementedError on a model sharded with the 2-way CFG split; it now lays the
    three branches out over the two halves (here: a loopback stand-in for the pair exchange, seen from each branch)."""
    from tests import fake_ops
    from viewcrafter_b200.ddim_multiplecond import DDIMSampler
    fake_ops.install(monkeypatch)
    model, x, c, uc, ui = _problem()
    seen = _record_batches(model)
    ref = _step(DDIMSampler(model, batch_cfg=True), x, c, uc, ui)

    class Loopback:
        """Both halves of the split in one process: the other branch's prediction is computed here, unsharded."""
        def __init__(self, branch, other):
            self.branch, self.other = branch, other

        def exchange(self, v_mine, rows=None):
            assert rows == (1, 2) and v_mine.shape[0] == rows[self.branch]
            return (v_mine, self.other) if self.branch == 0 else (self.other, v_mine)

    v_c, v_u, v_i = DDIMSampler(model, batch_cfg=True)._apply_stacked(x, torch.full((1,), 599), (c, uc, ui), {"fs": torch.tensor([10])})
    for branch, other in ((0, torch.cat([v_u, v_i], 0)), (1, v_c)):
        model._cfg = Loopback(branch, other)
        del seen[:]
        out = _step(DDIMSampler(model, batch_cfg=True), x, c, uc, ui)
        assert seen == ([(1, False)] if branch == 0 else [(2, True)])
        assert max(float((a - b).abs().max()) for a, b in zip(out, ref)) < 0.15


def _worker(rank, world, port, cfg_split, batch_cfg, T, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    import _pytest.monkeypatch as mpatch
    from tests import fake_ops
    from viewcrafter_b200 import parallel
    from viewcrafter_b200.ddim_multiplecond import DDIMSampler
    mpx = mpatch.MonkeyPatch()
    fake_ops.install(mpx)
    model, x, c, uc, ui = _problem(T)
    ref = _step(DDIMSampler(model, batch_cfg=batch_cfg), x, c, uc, ui)
    parallel.shard_model(model, dist, rank, world, cfg_split=cfg_split)
    assert (getattr(model, "_cfg", None) is not None) == cfg_split
    seen = _record_batches(model)
    out = _step(DDIMSampler(model, batch_cfg=batch_cfg), x, c, uc, ui)
    d = torch.tensor([max(float((a - b).abs().max()) for a, b in zip(out, ref))])
    dist.all_reduce(d, op=dist.ReduceOp.MAX)
    batches = [None] * world
    dist.all_gather_object(batches, seen)
    if rank == 0:
        q.put((float(d), batches))
    dist.barrier()
    dist.destroy_process_group()
    mpx.undo()


def _run(world, cfg_split, batch_cfg, T):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, cfg_split, batch_cfg, T, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=900)
        assert p.exitcode == 0, f"rank exited with {p.exitcode}"
    return q.get(timeout=10)


@pytest.mark.parametrize("world,batch_cfg", [(2, False), (2, True), (4, True), (8, True)])
def test_three_way_step_on_the_cfg_split_matches_single_process(world, batch_cfg):
    """Branch 0 (first half of the ranks) computes cond, branch 1 uncond + uncond_img; world 4 / 8 add 2- / 4-way frame sharding."""
    d, batches = _run(world, True, batch_cfg, 4)
    half = world // 2
    assert all(b == [(1, False)] for b in batches[:half]), batches
    branch1 = [(2, True)] if batch_cfg else [(1, False), (1, False)]
    assert all(b == branch1 for b in batches[half:]), batches
    # world 2 without batching runs the single-process forwards on each rank (identical); otherwise other batch sizes / frame
    # sharding change the fp16 roundings, which CFG amplifies ~16x
    assert d < (1e-5 if (world == 2 and not batch_cfg) else 0.15), d


@pytest.mark.parametrize("world,T", [(2, 4), (4, 5)])
def test_three_way_step_frame_sharded_matches_single_process(world, T):
    """cfg_split=False: the B=3 forward runs frame-sharded over all ranks (T=5 over 4 ranks: uneven frame ranges)."""
    d, batches = _run(world, False, True, T)
    assert all(b == [(3, True)] for b in batches), batches       # the prefix hint is passed, and ignored under frame sharding
    assert d < 0.15, d
