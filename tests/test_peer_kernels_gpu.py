"""The multi-GPU peer-memory kernels on ONE GPU, with every rank of the frame group emulated in one process (tests/peer_emul.py),
against exact layouts and float64 statistics.

Entry points: vc_peer_exchange (both directions, with the published GroupNorm sums), vc_peer_groupnorm_stats and
vc_peer_finish_scatter (gn_peer_allreduce_kernel), vc_peer_gather_leaves, the layout switch in the tap-GEMM epilogue
(vc_gemm_desc.peer: peer_scatter32) and vc_groupnorm_apply_parts.  The ranks run one after another on one stream, so what is checked
is every rank's routing, its published statistics, the slot parity and counters, graph capture, the grid-size independence and the
host-side refusals.  The cross-GPU memory ordering of the rendezvous (release / acquire over NVLink) is NOT exercised here.

Receive buffers are compared bit for bit (int16 views) with the slices FrameComm._to_sites / _to_frames define; NaN prefill and
guard rows catch missing and stray stores.  Statistics are held to an fp32 summation bound (peer_emul.sums_ratio) derived from the
depth of each kernel's summation tree; the GroupNorm outputs to the bounds of test_norm_statistics_gpu.py (section 7: the split form
this path replaces).  The worst error / bound per statistics path is printed at the end (run with -s).
"""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

from tests import peer_emul as pe
from tests.norm_rungs import REPORT, RUNGS, _gn_check, _note, affine, norm_ref, rung_data

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVEL = {9216: (72, 128, 320), 2304: (36, 64, 640), 576: (18, 32, 1280), 144: (9, 16, 1280)}    # U-Net levels at 576x1024: (H, W, C)


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from viewcrafter_b200 import ops as _ops
    return _ops


WORST = {}      # statistics path -> worst error / bound


def _worst(path, ratio):
    WORST[path] = max(WORST.get(path, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _report():
    REPORT.clear()
    yield
    if WORST:
        print("\nworst statistics error / fp32 summation bound per path (<= 1 passes)")
        for path, v in sorted(WORST.items()):
            print(f"  {path:44s} {v:.3g}")
    if REPORT:
        print("worst GroupNorm output error per rung (out/bound: |y - ref| / (3e-3 + 4e-3 |ref|); loose: |mean| > 64 std groups; rstd_rel: "
              "statistics from the gathered sums)")
        for (path, rung), d in sorted(REPORT.items()):
            print(f"  {path:28s} {rung:14s} " + " ".join(f"{k}={v:.3g}" for k, v in sorted(d.items())))


def make_x(B, T, HW, Cc, seed, offset=16.0):
    """fp16 [B, T, HW, C] = offset + N(0, 1): every row distinct with overwhelming probability, all sums well away from zero."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (offset + torch.randn(B, T, HW, Cc, generator=g, device="cuda")).half()


def assert_bits(got, want, what):
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} != {tuple(want.shape)}"
    g, w = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    if not torch.equal(g, w):
        bad = (g != w).any(1).nonzero()
        raise AssertionError(f"{what}: {bad.numel()} of {g.shape[0]} rows differ (first {bad[:4].flatten().tolist()}); "
                             f"NaN rows (never written): {int(torch.isnan(got.float()).any(1).sum())}")


# --------------------------------------------------------------------------------------------------- running one layout switch
def run_to_sites(grp, X, B, HW, order=None):
    """frames -> sites of the full X [B, T, HW, C] over every rank (with the published statistics)."""
    srcs = [pe.frames_of(X, grp.ranges, r) for r in range(grp.P)]
    for r in order or range(grp.P):
        grp.exchange(r, srcs[r], True, B, HW)
    return srcs


def run_to_frames(grp, X, B, HW):
    srcs = [pe.sites_of(X, grp.P, r) for r in range(grp.P)]
    for r in range(grp.P):
        grp.exchange(r, srcs[r], False, B, HW)
    return srcs


def check_sites(grp, X, bufs):
    for q in range(grp.P):
        assert_bits(bufs[q], pe.sites_of(X, grp.P, q), f"sites of rank {q}")


def check_frames(grp, X, bufs):
    for q in range(grp.P):
        assert_bits(bufs[q], pe.frames_of(X, grp.ranges, q), f"frames of rank {q}")


def slot_half(grp, q, B):
    s = int(grp.ranks[q].seq.item())
    return grp.ranks[q].slots[s & 1, :B]


def check_published(grp, parts, B, depth_of, path):
    """Every rank's slot half of the last collective holds all P ranks' (sum, sumsq), bit-identical across ranks; rank r's entry is
    within the fp32 summation bound of the float64 sums of parts[r] (rank r's rows, [B * n, C]).  Returns the slot half of rank 0."""
    half = slot_half(grp, 0, B)
    for q in range(1, grp.P):
        assert torch.equal(slot_half(grp, q, B).view(torch.int32), half.view(torch.int32)), f"{path}: slots of rank {q} != rank 0's"
    for r, x in enumerate(parts):
        ref, abss = pe.group_sums(x, B)
        _worst(path, pe.sums_ratio(half[:, r], ref, abss, depth_of(x.shape[0] // B, x.shape[1])))
    return half


def check_total(half, parts, B, depth_of):
    """The sums over the ranks (as vc_groupnorm_apply_parts combines them) against the float64 sums of all parts."""
    tot = half.double().sum(1)
    ref = sum(pe.group_sums(x, B)[0] for x in parts)
    abss = sum(pe.group_sums(x, B)[1] for x in parts)
    depth = max(depth_of(x.shape[0] // B, x.shape[1]) for x in parts) + len(parts)
    return pe.sums_ratio(tot.float(), ref, abss, depth)


# --------------------------------------------------------------------------------------------------- a. / b. the exchange kernel
EXCHANGE_CASES = [  # P, T, B, HW, C
    (2, 25, 1, 9216, 320), (2, 25, 3, 2304, 640), (2, 16, 4, 576, 1280), (2, 25, 2, 144, 1280), (2, 49, 1, 144, 1280),
    (3, 25, 1, 9216, 320), (3, 25, 2, 2304, 640), (3, 16, 4, 144, 1280), (3, 49, 3, 576, 1280),
    (4, 25, 1, 9216, 320), (4, 25, 4, 2304, 640), (4, 49, 2, 576, 1280), (4, 16, 3, 144, 1280),
    (8, 25, 1, 2304, 640), (8, 25, 3, 576, 1280), (8, 49, 2, 144, 1280), (8, 16, 4, 9216, 320),
    # C = 32 (128 rows per pass), 2560 and 4096 (one row per pass)
    (2, 25, 2, 576, 32), (8, 25, 4, 144, 32), (2, 25, 1, 144, 2560), (4, 16, 3, 576, 2560), (2, 25, 2, 144, 4096), (8, 25, 4, 144, 4096),
    # ranks with fewer rows than one pass of the 4-deep loop: the tail loop alone
    (8, 9, 1, 8, 32), (2, 3, 2, 16, 4096), (4, 5, 3, 32, 320),
]


@pytest.mark.parametrize("P,T,B,HW,Cc", EXCHANGE_CASES)
def test_exchange_routes_every_row_and_publishes_the_statistics(ops, P, T, B, HW, Cc):
    grp = pe.Group(P, T)
    X = make_x(B, T, HW, Cc, seed=P * 1000 + T * 10 + B)
    sites = grp.sites_buffers(B, Cc, HW)
    srcs = run_to_sites(grp, X, B, HW)
    check_sites(grp, X, sites)
    half = check_published(grp, srcs, B, pe.depth_exchange, "b exchange frames->sites")
    _worst("b exchange frames->sites (rank total)", check_total(half, srcs, B, pe.depth_exchange))
    last = grp.ranks[P - 1]
    assert torch.equal(last.cur_stats[:B].view(torch.int32), slot_half(grp, P - 1, B).view(torch.int32)), "cur_stats of the last rank"
    assert grp.state() == [(1, 0)] * P, "seq must advance by one and done return to 0"
    # and back: sites -> frames, no statistics
    frames = grp.frames_buffers(B, Cc, HW)
    run_to_frames(grp, X, B, HW)
    check_frames(grp, X, frames)
    assert grp.state() == [(2, 0)] * P
    grp.check_guards()


@pytest.mark.parametrize("P,T,B,HW,Cc", [(2, 25, 2, 576, 320), (3, 16, 1, 144, 1280), (4, 25, 3, 2304, 640), (8, 25, 4, 144, 320)])
def test_statistics_slots_alternate_and_the_last_rank_gathers(ops, P, T, B, HW, Cc):
    """P collectives, each with a different rank launched last and new data: the half (seq & 1) of every slot array is rewritten and
    complete, the other half is left alone, the last rank's cur_stats is a copy of its half, seq advances by one, done returns to 0."""
    grp = pe.Group(P, T)
    for k in grp.ranks:
        k.slots.fill_(float("nan"))
    sites = grp.sites_buffers(B, Cc, HW)
    for it in range(P):
        X = make_x(B, T, HW, Cc, seed=77 + it)
        last = it
        order = [(last + 1 + i) % P for i in range(P)]
        grp.refill("sites")
        srcs = run_to_sites(grp, X, B, HW, order=order)
        check_sites(grp, X, sites)
        assert grp.state() == [(it + 1, 0)] * P
        check_published(grp, srcs, B, pe.depth_exchange, "b exchange frames->sites")
        assert torch.equal(grp.ranks[last].cur_stats[:B].view(torch.int32), slot_half(grp, last, B).view(torch.int32)), f"iteration {it}"
        if it == 0:
            other = 1 - ((it + 1) & 1)
            assert all(bool(torch.isnan(k.slots[other]).all()) for k in grp.ranks), "the other parity half was written"
    grp.check_guards()


# --------------------------------------------------------------------------------------------------- c. peer GroupNorm statistics + apply
@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("P,T,B,HW,Cc,silu", [(2, 16, 2, 576, 320, True), (4, 25, 1, 144, 1280, False), (3, 7, 4, 48, 64, True)])
def test_peer_groupnorm_matches_float64_of_the_whole_tensor(ops, P, T, B, HW, Cc, silu, rung):
    """vc_peer_groupnorm_stats on every rank's site-layout rows, then vc_groupnorm_apply_parts: the normalised output of all ranks
    against float64 GroupNorm of the whole [B, T * HW, C] tensor, at section 7's bounds (including its 5 % rstd regression bound)."""
    eps = RUNGS[rung][0]
    X = rung_data(rung, B * T * HW, Cc, seed=91 + P, samples=B).view(B, T, HW, Cc)
    gamma, beta = affine(Cc, 8)
    grp = pe.Group(P, T)
    sites = [pe.sites_of(X, P, q) for q in range(P)]
    outs, stats = [None] * P, [None] * P
    for last in range(P):                      # a rank's gathered statistics are complete when it runs last
        for r in [(last + 1 + i) % P for i in range(P)]:
            grp.groupnorm_stats(r, sites[r], B)
        stats[last] = grp.ranks[last].cur_stats[:B].clone()
        outs[last] = grp.apply_parts(last, sites[last], B, T * HW, gamma, beta, eps, silu)
    assert grp.state() == [(P, 0)] * P
    for r in range(1, P):
        assert torch.equal(stats[r], stats[0]), f"rank {r} gathered other statistics than rank 0"
    out = pe.from_sites(outs, B, T).reshape(-1, Cc)
    _gn_check("c peer groupnorm", rung, out, X.reshape(-1, Cc), B, gamma, beta, eps, silu)
    st = stats[0].double().sum(1)
    n = T * HW * (Cc // 32)
    mean = st[..., 0] / n
    rstd = 1.0 / torch.sqrt((st[..., 1] / n - mean * mean).clamp_min(0.0) + eps)
    _, mean_ref, rstd_ref = norm_ref(X.reshape(-1, Cc), torch.ones(Cc, device="cuda"), torch.zeros(Cc, device="cuda"), eps, samples=B)
    rel = float(((rstd - rstd_ref) / rstd_ref).abs().max())
    _note("c peer groupnorm", rung, rstd_rel=rel, **{"mean*rstd": float(((mean - mean_ref).abs() * rstd_ref).max())})
    if not rung.startswith("const"):
        assert rel <= 0.05, f"peer statistics {rung}: rstd relative error {rel:.3g} (regression bound 5 %)"


# --------------------------------------------------------------------------------------------------- d. the layout switch in the GEMM epilogue
SCATTER_CASES = [  # producer, P, T, B, HW   (C from the level)
    ("conv3x3", 2, 25, 1, 9216), ("conv3x3", 2, 25, 3, 2304), ("conv3x3", 2, 16, 2, 576), ("conv3x3", 4, 25, 1, 9216),
    ("conv3x3", 4, 25, 2, 2304),
    ("linear_to_sites", 2, 25, 2, 9216), ("linear_to_sites", 2, 25, 1, 576), ("linear_to_sites", 4, 25, 3, 2304),
    ("linear_to_sites", 4, 16, 1, 9216),
    ("conv_temporal", 2, 25, 1, 9216), ("conv_temporal", 2, 25, 3, 2304), ("conv_temporal", 2, 16, 2, 576), ("conv_temporal", 4, 25, 2, 2304),
    ("conv_temporal", 4, 25, 1, 9216),
    ("linear_to_frames", 2, 25, 2, 9216), ("linear_to_frames", 2, 25, 1, 576), ("linear_to_frames", 4, 25, 3, 2304),
    ("linear_to_frames", 4, 16, 1, 9216),
]


def _weights(ops, producer, Cc, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if producer == "conv3x3":
        w = ops.pack_conv3x3(torch.randn(Cc, Cc, 3, 3, generator=g, device="cuda") / (3 * Cc ** 0.5))
    elif producer == "conv_temporal":
        w = ops.pack_conv_temporal(torch.randn(Cc, Cc, 3, 1, 1, generator=g, device="cuda") / (3 * Cc) ** 0.5)
    else:
        w = (torch.randn(Cc, Cc, generator=g, device="cuda") / Cc ** 0.5).half()
    return w, 0.1 * torch.randn(Cc, generator=g, device="cuda")


def run_scatter(ops, grp, producer, B, HW, w, bias, X, R, peer=True):
    """Every rank's GEMM on its rows of X (and residual R) with its output routed to the other layout (peer=True; then
    vc_peer_finish_scatter with the GEMM's GroupNorm records), or stored locally (peer=False).  Returns the GEMM outputs."""
    P, T, Cc = grp.P, grp.T, X.shape[3]
    H, W, _ = LEVEL[HW]
    outs = []
    for r in range(P):
        tl = grp.tl(r)
        plan = grp.plan(r, producer in ("conv3x3", "linear_to_sites"), B, HW, Cc) if peer else None
        if producer == "conv3x3":
            y = ops.conv3x3(pe.frames_of(X, grp.ranges, r), B * tl, H, W, w, bias=bias, res=pe.frames_of(R, grp.ranges, r), gn_out=True,
                            peer=plan)
        elif producer == "linear_to_sites":
            y = ops.linear(pe.frames_of(X, grp.ranges, r), w, bias=bias, res=pe.frames_of(R, grp.ranges, r), gn_out=True, peer=plan)
        elif producer == "conv_temporal":
            a = pe.sites_of(X, P, r)
            y = ops.conv_temporal(a, B, T, HW // P, w, bias=bias, res=a, peer=plan)          # the residual aliases the input (U-Net)
        else:
            a = pe.sites_of(X, P, r)
            y = ops.linear(a, w, bias=bias, res=a, peer=plan)
        if peer:
            geom = y.geom(B, tl * HW) if (plan.to_sites and y is not None) else None
            assert plan.to_sites == (geom is not None), "a frames -> sites switch must leave its GroupNorm records"
            grp.finish_scatter(r, geom, Cc, B)
        outs.append(y)
    return outs


@pytest.mark.parametrize("producer,P,T,B,HW", SCATTER_CASES)
def test_gemm_epilogue_scatter_equals_the_local_gemm_permuted(ops, producer, P, T, B, HW):
    Cc = LEVEL[HW][2]
    assert pe.scatter_case_ok(P, T, B, HW, Cc), "a shape the product never runs fused"
    grp = pe.Group(P, T)
    X = make_x(B, T, HW, Cc, seed=5 + P + B, offset=0.0)
    R = make_x(B, T, HW, Cc, seed=6 + P + B, offset=0.0)
    w, bias = _weights(ops, producer, Cc, seed=HW + P)
    to_sites = producer in ("conv3x3", "linear_to_sites")
    bufs = grp.sites_buffers(B, Cc, HW) if to_sites else grp.frames_buffers(B, Cc, HW)
    run_scatter(ops, grp, producer, B, HW, w, bias, X, R)
    local = run_scatter(ops, grp, producer, B, HW, w, bias, X, R, peer=False)
    if to_sites:
        Y = pe.from_frames(local, grp.ranges, B, HW)
        check_sites(grp, Y, bufs)
        depth = lambda rows, c: pe.depth_records(rows, c)     # noqa: E731
        half = check_published(grp, local, B, depth, "d gemm scatter records")
        _worst("d gemm scatter records (rank total)", check_total(half, local, B, depth))
        assert torch.equal(grp.ranks[P - 1].cur_stats[:B].view(torch.int32), slot_half(grp, P - 1, B).view(torch.int32))
    else:
        Y = pe.from_sites(local, B, T)
        check_frames(grp, Y, bufs)
    assert grp.state() == [(1, 0)] * P
    grp.check_guards()


# --------------------------------------------------------------------------------------------------- e. reproducible mode: the leaves
@pytest.mark.parametrize("P,T,B,HW,Cc", [(2, 25, 2, 576, 320), (4, 16, 1, 2304, 640), (8, 25, 3, 576, 1280), (8, 16, 1, 9216, 320)])
def test_gathered_leaves_are_the_single_gpu_leaves(ops, P, T, B, HW, Cc):
    """vc_peer_gather_leaves: the gathered array is torch.equal to groupnorm_leaves of the whole frame-layout tensor, and
    groupnorm_apply_leaves on each rank's sites equals the matching rows of single-GPU groupnorm_canonical (INTEGRATION.md)."""
    X = rung_data("mu16", B * T * HW, Cc, seed=P + HW, samples=B).view(B, T, HW, Cc)
    gamma, beta = affine(Cc, 9)
    nc = ops.gn_leaf_chunks(HW)
    assert nc % P == 0
    full = X.reshape(-1, Cc)
    want = ops.groupnorm_leaves(full, HW // nc)
    canon = ops.groupnorm_canonical(full, B, HW, gamma, beta, 1e-5, True).view(B, T, HW, Cc)
    grp = pe.Group(P, T)
    grp.leaf_buffers(B * T * nc * 64)
    sites = [pe.sites_of(X, P, q) for q in range(P)]
    leaves = [ops.groupnorm_leaves(s, HW // nc) for s in sites]
    for last in range(P):
        grp.refill_leaves()
        got = [torch.full((B * T * nc, 32, 2), float("nan"), device="cuda") for _ in range(P)]
        for r in [(last + 1 + i) % P for i in range(P)]:
            grp.gather_leaves(r, leaves[r], B, nc, got[r])
        assert torch.equal(got[last], want), f"rank {last}: gathered leaves differ from the single-GPU leaves"
        out = ops.groupnorm_apply_leaves(sites[last], B, got[last], T * HW, gamma, beta, 1e-5, True)
        assert torch.equal(out, pe.sites_of(canon, P, last)), f"rank {last}: apply_leaves differs from groupnorm_canonical"
    assert grp.state() == [(P, 0)] * P
    grp.check_guards()


# --------------------------------------------------------------------------------------------------- f. CUDA-graph replay
GRAPH_SCATTER = ("conv3x3", 2, 25, 2, 2304)


def _graph_case(ops, kind):
    if kind == "exchange":
        P, T, B, HW, Cc = 4, 25, 2, 2304, 640
    else:
        _, P, T, B, HW = GRAPH_SCATTER
        Cc = LEVEL[HW][2]
    groups = [pe.Group(P, T), pe.Group(P, T)]                   # [graph, eager]: the same collective sequence on separate state
    bufs = [g.sites_buffers(B, Cc, HW) for g in groups]
    w, bias = _weights(ops, "conv3x3", Cc, seed=3)
    X = [make_x(B, T, HW, Cc, seed=1, offset=0.0) for _ in groups]
    R = [make_x(B, T, HW, Cc, seed=2, offset=0.0) for _ in groups]
    srcs = [[pe.frames_of(x, g.ranges, r) for r in range(P)] for x, g in zip(X, groups)]
    keep = []

    def run(i):
        g = groups[i]
        if kind == "exchange":
            for r in range(P):
                g.exchange(r, srcs[i][r], True, B, HW)
        else:
            keep.append(run_scatter(ops, g, "conv3x3", B, HW, w, bias, X[i], R[i]))
    return groups, bufs, X, R, srcs, run, (P, T, B, HW, Cc)


@pytest.mark.parametrize("kind", ["exchange", "scatter"])
def test_graph_replay_equals_eager(ops, kind):
    groups, bufs, X, R, srcs, run, (P, T, B, HW, Cc) = _graph_case(ops, kind)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(0)
    torch.cuda.current_stream().wait_stream(s)
    run(1)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run(0)
    parities = []
    for it in range(3):
        Xn, Rn = make_x(B, T, HW, Cc, seed=40 + it, offset=0.0), make_x(B, T, HW, Cc, seed=50 + it, offset=0.0)
        for i, g in enumerate(groups):
            X[i].copy_(Xn)
            R[i].copy_(Rn)
            for r in range(P):
                srcs[i][r].copy_(pe.frames_of(Xn, g.ranges, r))
            g.refill("sites")
        graph.replay()
        run(1)
        torch.cuda.synchronize()
        for q in range(P):
            assert torch.equal(bufs[0][q].view(torch.int16), bufs[1][q].view(torch.int16)), f"replay {it}: sites of rank {q}"
        sg, se = groups[0].state(), groups[1].state()
        assert sg == se and sg[0][0] == it + 2, (sg, se)
        parities.append(sg[0][0] & 1)
        for q in range(P):
            assert torch.equal(slot_half(groups[0], q, B).view(torch.int32), slot_half(groups[1], q, B).view(torch.int32)), f"replay {it}"
        assert torch.equal(groups[0].ranks[P - 1].cur_stats[:B], groups[1].ranks[P - 1].cur_stats[:B])
        if kind == "exchange":
            check_sites(groups[0], Xn, bufs[0])
            check_published(groups[0], srcs[0], B, pe.depth_exchange, "f graph exchange")
    assert parities == [0, 1, 0]
    for g in groups:
        g.check_guards()


# --------------------------------------------------------------------------------------------------- g. refusals before any launch
def _refused(ops, fn):
    n0 = ops.launch_count()
    with pytest.raises(ops.VcError):
        fn()
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, "a refused call launched a kernel"


def test_refusals_launch_nothing(ops):
    P, T, B, HW, Cc = 2, 4, 1, 64, 64
    grp = pe.Group(P, T)
    grp.sites_buffers(4, 4096, HW)
    grp.frames_buffers(4, 4096, HW)
    k = grp.ranks[0]
    src = torch.zeros((4 * T * HW, 4096), dtype=torch.float16, device="cuda")

    def ex(r=0, B=B, HW=HW, Cc=Cc, f0=None, dst=None, g=grp, to_sites=1, comm=None):
        g.launch(r, "vc_peer_exchange", src.data_ptr(), dst or g.ptrs("sites"), to_sites, B, g.T, HW, Cc, g.f0_arr(f0), 1,
                 g.ranks[r].ws.data_ptr(), g.ranks[r].ws.numel() * 4, comm=comm)

    _refused(ops, lambda: ex(B=5))                                   # B > Bmax
    small = pe.Group(P, T, bmax=2)
    small.sites_buffers(4, Cc, HW)
    _refused(ops, lambda: ex(B=3, g=small))                          # B > Bmax of a Bmax = 2 group
    _refused(ops, lambda: ex(HW=63))                                 # HW % P
    _refused(ops, lambda: ex(Cc=48))                                 # C % 32
    _refused(ops, lambda: ex(Cc=4128))                               # C > 4096
    _refused(ops, lambda: ex(f0=[0, 2, 3]))                          # ranges end before T
    _refused(ops, lambda: ex(f0=[1, 2, 4]))                          # ... or start after 0
    _refused(ops, lambda: ex(dst=(C.c_void_p * P)(grp.ranks[0].bufs["sites"][0].data_ptr(), None)))   # null destination
    empty = pe.Group(4, 3)                                           # frame ranges 1/1/1/0: rank 3 owns no frames
    empty.sites_buffers(1, Cc, HW)
    _refused(ops, lambda: ex(r=3, g=empty))
    for field, val in (("world", 9), ("world", 0), ("rank", 2), ("rank", -1), ("Bmax", 0), ("Bmax", 5)):
        bad = type(grp.comms[0]).from_buffer_copy(grp.comms[0])
        setattr(bad, field, val)
        _refused(ops, lambda: ex(comm=bad))
    x = src[:B * T * HW, :Cc]
    _refused(ops, lambda: grp.launch(0, "vc_peer_groupnorm_stats", x.data_ptr(), Cc, 5, T * HW, k.ws.data_ptr(), k.ws.numel() * 4))
    geom = ops.GnPartGeom()
    _refused(ops, lambda: grp.launch(0, "vc_peer_finish_scatter", C.byref(geom), Cc, 5, k.ws.data_ptr(), k.ws.numel() * 4))
    cap = grp.leaf_buffers(B * T * 8 * 64)
    leaves = torch.zeros((B * T * 8, 32, 2), device="cuda")
    out = torch.empty_like(leaves)
    lptrs = (C.c_void_p * P)(*[q.leaves[0].data_ptr() for q in grp.ranks])
    _refused(ops, lambda: grp.launch(0, "vc_peer_gather_leaves", leaves.data_ptr(), lptrs, cap, B, T, 3, out.data_ptr()))      # nc % P
    _refused(ops, lambda: grp.launch(0, "vc_peer_gather_leaves", leaves.data_ptr(), lptrs, B * T * 8 * 64 - 1, B, T, 8, out.data_ptr()))
    # the GEMM epilogue takes at most 4 ranks
    g8 = pe.Group(8, 8)
    g8.sites_buffers(1, 32, 256)
    xg = torch.zeros((256, 32), dtype=torch.float16, device="cuda")
    _refused(ops, lambda: ops.linear(xg, torch.zeros((32, 32), dtype=torch.float16, device="cuda"), peer=g8.plan(0, True, 1, 256, 32)))
    assert grp.state() == [(0, 0)] * P, "a refused collective advanced the sequence"
    n0 = ops.launch_count()                                          # and the counter does see the launches it must not see above
    for r in range(P):
        ex(r=r)
    assert ops.launch_count() == n0 + P and grp.state() == [(1, 0)] * P


# --------------------------------------------------------------------------------------------------- h. grid size
GRID_EXCHANGE = [(2, 25, 1, 9216, 320), (4, 25, 3, 2304, 640), (3, 49, 2, 144, 1280), (8, 16, 4, 576, 32)]
GRID_SCATTER = [("conv3x3", 2, 25, 2, 2304), ("conv_temporal", 2, 25, 1, 576), ("linear_to_sites", 4, 25, 1, 9216)]


def grid_cases():
    """Receive buffers and gathered statistics of a fixed set of exchanges and epilogue scatters (run in this process, and in a child
    whose launch grids are cut by VC_SM_COUNT)."""
    from viewcrafter_b200 import ops
    res = {}
    for P, T, B, HW, Cc in GRID_EXCHANGE:
        grp = pe.Group(P, T)
        X = make_x(B, T, HW, Cc, seed=HW + Cc)
        bufs = grp.sites_buffers(B, Cc, HW)
        run_to_sites(grp, X, B, HW)
        res[f"exchange {P} {T} {B} {HW} {Cc}"] = {"bufs": torch.stack(bufs).cpu(), "stats": slot_half(grp, 0, B).cpu()}
        grp.groupnorm_stats(P - 1, bufs[P - 1], B)             # peer_groupnorm_stats: rank P - 1's part, published to rank 0's slots
        half = int(grp.ranks[P - 1].seq.item()) & 1
        res[f"exchange {P} {T} {B} {HW} {Cc}"]["gn_stats"] = grp.ranks[0].slots[half, :B, P - 1].cpu()
    for producer, P, T, B, HW in GRID_SCATTER:
        Cc = LEVEL[HW][2]
        grp = pe.Group(P, T)
        X = make_x(B, T, HW, Cc, seed=11, offset=0.0)
        R = make_x(B, T, HW, Cc, seed=12, offset=0.0)
        w, bias = _weights(ops, producer, Cc, seed=13)
        to_sites = producer in ("conv3x3", "linear_to_sites")
        bufs = grp.sites_buffers(B, Cc, HW) if to_sites else grp.frames_buffers(B, Cc, HW)
        run_scatter(ops, grp, producer, B, HW, w, bias, X, R)
        d = {"bufs": [b.cpu() for b in bufs]}
        if to_sites:
            d["stats"] = slot_half(grp, 0, B).cpu()
        res[f"scatter {producer} {P} {T} {B} {HW}"] = d
    torch.cuda.synchronize()
    return res


def grid_main(path):
    torch.save(grid_cases(), path)
    print("PEER_GRID_OK")


def test_results_do_not_depend_on_the_grid_size(ops, tmp_path):
    """A child process with VC_SM_COUNT=3 (every launch grid sized for 3 SMs): receive buffers bit-identical to this process's full
    grid, statistics within their fp32 summation bound of float64."""
    full = grid_cases()
    env = dict(os.environ, VC_SM_COUNT="3")
    env.pop("VC_REPRODUCIBLE", None)
    path = tmp_path / "grid3.pt"
    p = subprocess.run([sys.executable, "-c", "import sys; from tests import test_peer_kernels_gpu as m; m.grid_main(sys.argv[1])", str(path)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    print(p.stdout[-3000:])
    assert p.returncode == 0 and "PEER_GRID_OK" in p.stdout
    got = torch.load(path)
    assert sorted(got) == sorted(full)
    for name, d in full.items():
        bufs_g, bufs_f = got[name]["bufs"], d["bufs"]
        for q, (a, b) in enumerate(zip(bufs_g, bufs_f)):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"VC_SM_COUNT=3: {name}: receive buffer of rank {q}"
    # statistics of the small grid against float64
    for P, T, B, HW, Cc in GRID_EXCHANGE:
        name = f"exchange {P} {T} {B} {HW} {Cc}"
        X = make_x(B, T, HW, Cc, seed=HW + Cc)
        ranges = pe.parallel.frame_ranges(T, P)
        for r in range(P):
            ref, abss = pe.group_sums(pe.frames_of(X, ranges, r), B)
            depth = pe.depth_exchange((ranges[r][1] - ranges[r][0]) * HW, Cc)
            _worst("h exchange, 3-SM grid", pe.sums_ratio(got[name]["stats"][:, r].cuda(), ref, abss, depth))
        ref, abss = pe.group_sums(pe.sites_of(X, P, P - 1), B)
        # gn_stats_kernel: per-thread runs, the CTA's ppi * cg sums and the splits are no longer than the exchange kernel's
        _worst("h peer_groupnorm_stats, 3-SM grid", pe.sums_ratio(got[name]["gn_stats"].cuda(), ref, abss, pe.depth_exchange(T * (HW // P), Cc)))
    for producer, P, T, B, HW in GRID_SCATTER:
        if producer not in ("conv3x3", "linear_to_sites"):
            continue
        Cc = LEVEL[HW][2]
        grp = pe.Group(P, T)
        w, bias = _weights(ops, producer, Cc, seed=13)
        local = run_scatter(ops, grp, producer, B, HW, w, bias, make_x(B, T, HW, Cc, seed=11, offset=0.0), make_x(B, T, HW, Cc, seed=12, offset=0.0),
                            peer=False)
        for r, y in enumerate(local):
            ref, abss = pe.group_sums(y, B)
            _worst("h gemm scatter records, 3-SM grid", pe.sums_ratio(got[f"scatter {producer} {P} {T} {B} {HW}"]["stats"][:, r].cuda(), ref, abss,
                                                                      pe.depth_records(y.shape[0] // B, Cc)))


# --------------------------------------------------------------------------------------------------- i. negative controls (reference side)
def test_the_checks_catch_wrong_routes_statistics_and_leaves(ops):
    """Mutations of the REFERENCE, applied to real kernel outputs: each must fall outside the checks above."""
    P, T, B, HW, Cc = 4, 25, 2, 576, 320
    grp = pe.Group(P, T)
    X = make_x(B, T, HW, Cc, seed=123)
    sites = grp.sites_buffers(B, Cc, HW)
    srcs = run_to_sites(grp, X, B, HW)
    check_sites(grp, X, sites)
    want = [pe.sites_of(X, P, q) for q in range(P)]
    with pytest.raises(AssertionError):                      # a route off by one row
        assert_bits(sites[1], torch.roll(want[1], 1, 0), "off by one")
    with pytest.raises(AssertionError):                      # two ranks swapped
        assert_bits(sites[0], want[1], "swapped")
    half = check_published(grp, srcs, B, pe.depth_exchange, "i control")
    check_total(half, srcs, B, pe.depth_exchange)
    with pytest.raises(AssertionError):                      # statistics missing one rank
        check_total(half, srcs[1:], B, pe.depth_exchange)
    with pytest.raises(AssertionError):                      # one rank's statistics credited to another
        ref, abss = pe.group_sums(srcs[1], B)
        pe.sums_ratio(half[:, 0], ref, abss, pe.depth_exchange(srcs[0].shape[0] // B, Cc))
    # leaves with one chunk misplaced
    nc = ops.gn_leaf_chunks(HW)
    full = X.reshape(-1, Cc)
    want_l = ops.groupnorm_leaves(full, HW // nc)
    grp.leaf_buffers(B * T * nc * 64)
    got = [torch.empty_like(want_l) for _ in range(P)]
    for r in range(P):
        grp.gather_leaves(r, ops.groupnorm_leaves(want[r], HW // nc), B, nc, got[r])
    assert torch.equal(got[P - 1], want_l)
    moved = want_l.clone()
    moved[[0, 1]] = want_l[[1, 0]]
    assert not torch.equal(got[P - 1], moved), "a misplaced chunk went unnoticed"
    grp.check_guards()
