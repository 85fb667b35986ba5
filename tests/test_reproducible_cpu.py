"""Host logic of reproducible mode with the CPU double of the kernels (tests/fake_ops.py) and gloo: the switch, its route to the
GroupNorm leaves and into the CUDA-graph key, the site-layout 5-D GroupNorm over 2 and 4 ranks (bit-identical to one process), and
shard_model's checks."""
import multiprocessing as mp
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

from viewcrafter_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- CPU double of the leaf kernels: per-leaf sums in a fixed order, index-order fp64 combine (see test_gn_leaves_model_cpu.py) ----
calls = []


def fake_groupnorm_leaves(x, rows_per_leaf, x2=None):
    a = (x if x2 is None else torch.cat([x, x2], 1)).float()
    calls.append(("leaves", a.shape[0], rows_per_leaf))
    blocks = a.reshape(-1, rows_per_leaf, 32, a.shape[1] // 32)
    return torch.stack([torch.stack([b.sum((0, 2)), (b * b).sum((0, 2))], -1) for b in blocks]).contiguous()


def fake_groupnorm_apply_leaves(x, samples, leaves, stat_rows, gamma, beta, eps, silu, x2=None):
    from tests import fake_ops
    calls.append(("apply", samples, leaves.shape[0] // samples, stat_rows))
    lv = leaves.double().reshape(samples, -1, 32, 2)
    acc = torch.zeros((samples, 32, 2), dtype=torch.float64)
    for i in range(lv.shape[1]):
        acc += lv[:, i]
    a = x if x2 is None else torch.cat([x, x2], 1)
    return fake_ops.groupnorm_apply(a, samples, acc.float(), stat_rows, gamma, beta, eps, silu)


def install_leaves(monkeypatch):
    monkeypatch.setattr(ops, "groupnorm_leaves", fake_groupnorm_leaves)
    monkeypatch.setattr(ops, "groupnorm_apply_leaves", fake_groupnorm_apply_leaves)


@pytest.fixture
def repro():
    prev = ops.set_reproducible(True)
    yield
    ops.set_reproducible(prev)


def test_switch_and_environment():
    prev = ops.set_reproducible(True)
    try:
        import viewcrafter_b200
        assert viewcrafter_b200.reproducible() and ops.set_reproducible(False) is True and not ops.reproducible()
    finally:
        ops.set_reproducible(prev)
    code = "import viewcrafter_b200 as v; print(v.reproducible())"
    for val, want in (("1", "True"), ("0", "False")):
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, env=dict(os.environ, VC_REPRODUCIBLE=val))
        assert r.stdout.strip() == want, r.stderr


def test_groupnorm_routes_to_leaves(monkeypatch, repro):
    install_leaves(monkeypatch)
    calls.clear()
    x = torch.randn(3 * 160, 64).half()
    g, b = torch.ones(64), torch.zeros(64)
    ops.groupnorm(x, 3, g, b, 1e-5, True)                          # per frame: 3 frames of 160 pixels, nc = 8
    ops.groupnorm_canonical(x, 1, 160, g, b, 1e-5, True)           # 5-D: one sample of 3 frames
    assert calls == [("leaves", 480, 20), ("apply", 3, 8, 160), ("leaves", 480, 20), ("apply", 1, 24, 480)]
    assert not ops._want_gn(True, 100)                              # no producer sums are requested in this mode
    ops.set_reproducible(False)
    assert ops._want_gn(True, 100) == (ops.GN_FROM_PRODUCER >= 1)


def test_unet_forward_takes_every_groupnorm_from_leaves(monkeypatch, repro):
    from oracle import synth
    from tests import fake_ops
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    real_gn = ops.groupnorm
    fake_ops.install(monkeypatch)
    monkeypatch.setattr(ops, "groupnorm", real_gn)                 # the real dispatcher, with the CPU double of the leaf kernels
    install_leaves(monkeypatch)
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64)).eval()
    m.load_state_dict(synth.synth_state_dict(synth.module_shapes(m), 5), strict=True)
    T, H, W = 3, 16, 16
    x = torch.randn(1, 8, T, H, W)
    calls.clear()
    y = m(x, torch.tensor([499]), context=torch.randn(1, 333, 1024), fs=torch.tensor([10]))
    assert torch.isfinite(y).all()
    applies = [c for c in calls if c[0] == "apply"]
    five_d = [c for c in applies if c[1] == 1]                      # one sample of T frames: TemporalConvBlock / TemporalTransformer
    per_frame = [c for c in applies if c[1] == T]
    assert five_d and per_frame and len(five_d) + len(per_frame) == len(applies)
    for _, _, per_sample, stat_rows in five_d:
        hw = stat_rows // T
        assert per_sample == T * ops.gn_leaf_chunks(hw)
    for _, _, per_sample, stat_rows in per_frame:
        assert per_sample == ops.gn_leaf_chunks(stat_rows)


def test_graph_key_includes_the_mode(monkeypatch):
    from viewcrafter_b200.configs import UNET_PARAMS
    from viewcrafter_b200.unet import UNetModel
    m = UNetModel(**dict(UNET_PARAMS, model_channels=64))
    monkeypatch.setattr(m, "_forward_impl", lambda *a, **k: None)
    ctx = torch.zeros(1, 4)
    prev = ops.set_reproducible(False)
    try:
        m._forward_graphed(torch.zeros(1, 8, 1, 8, 8), torch.zeros(1), ctx, None, {})
        ops.set_reproducible(True)
        m._forward_graphed(torch.zeros(1, 8, 1, 8, 8), torch.zeros(1), ctx, None, {})
    finally:
        ops.set_reproducible(prev)
    keys = list(m._graphs)
    assert len(keys) == 2 and {k[-1] for k in keys} == {False, True}


# ---- multi-process (gloo) ----
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _run(target, world, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q) + args) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0, f"rank exited with {p.exitcode}"
    return [q.get(timeout=10) for _ in range(world)]


def _gn5d_worker(rank, world, port, q, B):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    import _pytest.monkeypatch as mpatch
    from viewcrafter_b200 import parallel
    mpx = mpatch.MonkeyPatch()
    install_leaves(mpx)
    ops.set_reproducible(True)
    T, HW, C = 25, 160, 64
    g = torch.Generator().manual_seed(B)
    x = (torch.randn(B, T, HW, C, generator=g) * 1.5 + 0.3).half()
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    single = ops.groupnorm_canonical(x.reshape(-1, C), B, HW, gamma, beta, 1e-5, True).reshape(B, T, HW, C)
    comm = parallel.FrameComm(dist, rank, world)
    comm.bind(T)
    HWl = HW // world
    mine = x[:, :, rank * HWl:(rank + 1) * HWl].reshape(-1, C).contiguous()
    y = comm.groupnorm5d(mine, B, gamma, beta, 1e-5, True, T * HW, fresh=True)
    q.put(bool(torch.equal(y, single[:, :, rank * HWl:(rank + 1) * HWl].reshape(-1, C))))
    dist.barrier()
    dist.destroy_process_group()
    mpx.undo()


@pytest.mark.parametrize("world,B", [(2, 1), (2, 3), (4, 2)])
def test_site_layout_groupnorm_is_bit_identical_to_one_process(world, B):
    assert all(_run(_gn5d_worker, world, B))


def _shard_worker(rank, world, port, q, modes, cfg_split):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from viewcrafter_b200 import parallel
    ops.set_reproducible(modes[rank])
    try:
        parallel.shard_model(torch.nn.Linear(2, 2), dist, rank, world, cfg_split=cfg_split)
        q.put("ok")
    except (ValueError, RuntimeError) as e:
        q.put(type(e).__name__ + ": " + str(e))
    dist.destroy_process_group()


def test_shard_model_checks():
    out = _run(_shard_worker, 2, (True, False), False)
    assert all("disagree on reproducible mode" in o for o in out), out
    out = _run(_shard_worker, 3, (True, True, True), False)
    assert all("frame groups of 1, 2, 4 or 8" in o for o in out), out
    out = _run(_shard_worker, 2, (True, True), False)
    assert out == ["ok", "ok"]
