"""Every rank of a frame group of P ranks, emulated in one process on one GPU, for the peer-memory kernels (csrc/peer.cu and the
layout switch in the tap-GEMM epilogue).

The kernels store through pointers, and those may point at buffers on the same device, so each rank gets plain device tensors (flag
words, sequence and completion counters, statistics slots, workspace, receive buffers) and a `_lib.PeerComm` whose peer pointers are
the other emulated ranks' tensors.  No IPC, no process group.  The ranks run one after another on one stream.  Their only cross-rank
dependency is the rendezvous in peer_finish: rank r waits until flags_r[q] >= seq_r + 1 for every q.  `Group.launch` satisfies it
before the launch by storing seq_r + 1 into all of flags_r, on the same stream (so also inside a captured CUDA graph): the kernel
computes its target from the same counter and never enters the wait loop.  Every vc_peer_* call goes through `Group.launch`.

What sequential emulation cannot give: a rank's gathered statistics (cur_stats) and gathered leaves are complete only when it runs
last, after every peer has published.  The tests therefore rotate which rank runs last.  The cross-GPU memory ordering of the protocol
is not exercised at all.

Receive buffers are NaN where data must land and are followed by GUARD rows of a sentinel, so a store outside its range shows as a
changed guard (`Group.check_guards`) instead of a corrupted neighbour.
"""
import ctypes as C

import torch

from viewcrafter_b200 import _lib, parallel

NAN16 = 0x7E00            # fp16 quiet NaN
SENT16 = 0x5A5A           # fp16 sentinel of the guard rows (203.25)
SENT32 = 0x5A5A5A5A       # float32 sentinel of the leaf guards
GUARD = 64                # guard rows after every receive buffer


def _fill16(t: torch.Tensor, bits: int):
    t.view(torch.int16).fill_(bits)


class _Rank:
    def __init__(self, P: int, bmax: int, dev):
        self.flags = torch.zeros(P, dtype=torch.int32, device=dev)
        self.seq = torch.zeros(1, dtype=torch.int32, device=dev)
        self.done = torch.zeros(1, dtype=torch.int32, device=dev)
        self.slots = torch.zeros((2, bmax, P, 32, 2), dtype=torch.float32, device=dev)
        self.cur_stats = torch.zeros((bmax, P, 32, 2), dtype=torch.float32, device=dev)
        self.ws = torch.empty(bmax * 512 * 64, dtype=torch.float32, device=dev)
        self.bufs = {}        # name -> (tensor of rows + GUARD rows, data rows)
        self.leaves = None    # (float32 [2, cap], cap, n): n leaf floats, then guards, per half


class Group:
    """P emulated ranks of a frame group over T frames (frame ranges: parallel.frame_ranges)."""

    def __init__(self, P: int, T: int, bmax: int = 4, device="cuda"):
        self.lib = _lib.load()
        self.P, self.T, self.bmax = P, T, bmax
        self.ranges = parallel.frame_ranges(T, P)
        self.f0 = [r[0] for r in self.ranges] + [T]
        self.ranks = [_Rank(P, bmax, device) for _ in range(P)]
        self.comms = []
        for r, k in enumerate(self.ranks):
            c = _lib.PeerComm()
            c.world, c.rank, c.Bmax = P, r, bmax
            c.flags, c.seq, c.done, c.cur_stats = k.flags.data_ptr(), k.seq.data_ptr(), k.done.data_ptr(), k.cur_stats.data_ptr()
            for q in range(P):
                c.peer_flags[q] = self.ranks[q].flags.data_ptr()
                c.stats_slots[q] = self.ranks[q].slots.data_ptr()
            self.comms.append(c)

    def tl(self, r: int) -> int:
        return self.ranges[r][1] - self.ranges[r][0]

    # -- the one way a collective is launched -------------------------------------------------------------------------------------
    def launch(self, r: int, entry: str, *args, comm=None):
        """Rank r's collective: lib.<entry>(comm of rank r, *args, stream), after flags_r[:] = seq_r + 1 on the same stream.
        `comm`: a (deliberately malformed) PeerComm to pass instead of rank r's."""
        k = self.ranks[r]
        k.flags.copy_((k.seq + 1).expand(self.P))
        c = self.comms[r] if comm is None else comm
        _lib.check(getattr(self.lib, entry)(C.byref(c), *args, torch.cuda.current_stream().cuda_stream), entry)

    # -- receive buffers ----------------------------------------------------------------------------------------------------------
    def buffer(self, r: int, name: str, rows: int, Cc: int) -> torch.Tensor:
        """Rank r's fp16 receive buffer `name` of rows x Cc (+ GUARD rows), NaN-filled, guards set.  Returns the data rows."""
        full = torch.empty(((rows + GUARD) * Cc,), dtype=torch.float16, device=self.ranks[r].flags.device)
        _fill16(full[:rows * Cc], NAN16)
        _fill16(full[rows * Cc:], SENT16)
        self.ranks[r].bufs[name] = (full, rows * Cc)
        return full[:rows * Cc].view(rows, Cc)

    def sites_buffers(self, B: int, Cc: int, HW: int):
        return [self.buffer(q, "sites", B * self.T * (HW // self.P), Cc) for q in range(self.P)]

    def frames_buffers(self, B: int, Cc: int, HW: int):
        return [self.buffer(q, "frames", B * self.tl(q) * HW, Cc) for q in range(self.P)]

    def refill(self, name: str):
        """NaN into the data rows of every rank's buffer `name` again (guards untouched)."""
        for k in self.ranks:
            full, n = k.bufs[name]
            _fill16(full[:n], NAN16)

    def leaf_buffers(self, n: int):
        """Every rank's float32 leaf buffer [2][cap], cap = n + GUARD * 64: both halves NaN over [0, n), sentinel over [n, cap)."""
        cap = n + GUARD * 64
        for k in self.ranks:
            t = torch.empty((2, cap), dtype=torch.float32, device=k.flags.device)
            k.leaves = (t, cap, n)
        self.refill_leaves()
        return cap

    def refill_leaves(self):
        for k in self.ranks:
            t, cap, n = k.leaves
            t[:, :n].fill_(float("nan"))
            t[:, n:].view(torch.int32).fill_(SENT32)

    def check_guards(self):
        for r, k in enumerate(self.ranks):
            for name, (full, n) in k.bufs.items():
                assert bool((full[n:].view(torch.int16) == SENT16).all()), f"rank {r}: guard of '{name}' overwritten"
            if k.leaves is not None:
                t, cap, n = k.leaves
                assert bool((t[:, n:].view(torch.int32) == SENT32).all()), f"rank {r}: leaf guard overwritten"

    def ptrs(self, name: str):
        return (C.c_void_p * self.P)(*[k.bufs[name][0].data_ptr() for k in self.ranks])

    def f0_arr(self, f0=None):
        f0 = self.f0 if f0 is None else f0
        return (C.c_int32 * len(f0))(*f0)

    # -- the collectives ------------------------------------------------------------------------------------------------------------
    def exchange(self, r: int, src: torch.Tensor, to_sites: bool, B: int, HW: int, with_stats: bool = True):
        """vc_peer_exchange of rank r (frames -> sites into the 'sites' buffers, or sites -> frames into 'frames')."""
        k = self.ranks[r]
        self.launch(r, "vc_peer_exchange", src.data_ptr(), self.ptrs("sites" if to_sites else "frames"), int(to_sites), B, self.T, HW,
                    src.shape[1], self.f0_arr(), int(with_stats), k.ws.data_ptr(), k.ws.numel() * 4)

    def groupnorm_stats(self, r: int, x: torch.Tensor, B: int):
        k = self.ranks[r]
        self.launch(r, "vc_peer_groupnorm_stats", x.data_ptr(), x.shape[1], B, x.shape[0] // B, k.ws.data_ptr(), k.ws.numel() * 4)

    def finish_scatter(self, r: int, geom, Cc: int, B: int):
        k = self.ranks[r]
        self.launch(r, "vc_peer_finish_scatter", C.byref(geom) if geom is not None else None, Cc, B, k.ws.data_ptr(), k.ws.numel() * 4)

    def gather_leaves(self, r: int, leaves: torch.Tensor, B: int, nc: int, out: torch.Tensor):
        cap = self.ranks[0].leaves[1]
        self.launch(r, "vc_peer_gather_leaves", leaves.data_ptr(), (C.c_void_p * self.P)(*[k.leaves[0].data_ptr() for k in self.ranks]),
                    cap, B, self.T, nc, out.data_ptr())

    def apply_parts(self, r: int, x: torch.Tensor, B: int, stat_rows: int, gamma, beta, eps: float, silu: bool) -> torch.Tensor:
        """vc_groupnorm_apply_parts with rank r's gathered statistics (a local kernel: no rendezvous)."""
        out = torch.empty_like(x)
        _lib.check(self.lib.vc_groupnorm_apply_parts(x.data_ptr(), x.shape[1], B, x.shape[0] // B, self.ranks[r].cur_stats.data_ptr(), self.P,
                                                     stat_rows, gamma.data_ptr(), beta.data_ptr(), eps, int(silu), out.data_ptr(),
                                                     torch.cuda.current_stream().cuda_stream), "vc_groupnorm_apply_parts")
        return out

    def plan(self, r: int, to_sites: bool, B: int, HW: int, Cc: int):
        return Plan(self, r, to_sites, B, HW, Cc)

    def state(self):
        """(seq, done) of every rank, on the host."""
        return [(int(k.seq.item()), int(k.done.item())) for k in self.ranks]


class Plan:
    """parallel._ScatterPlan for one emulated rank: attach() routes the GEMM's output tiles into the emulated ranks' receive buffers
    exactly as _ScatterPlan.attach does; finish() returns the GEMM's GroupNorm records (the test then runs vc_peer_finish_scatter)."""

    def __init__(self, group: Group, r: int, to_sites: bool, B: int, HW: int, Cc: int):
        self.to_sites, self.B, self.HW, self.C = to_sites, B, HW, Cc
        P, T = group.P, group.T
        self.rows_in = B * group.tl(r) * HW if to_sites else B * T * (HW // P)
        name = "sites" if to_sites else "frames"
        self.own = group.ranks[r].bufs[name][0]
        g = _lib.GemmPeer()
        g.mode, g.world, g.rank, g.B, g.T, g.HW = (1 if to_sites else 2), P, r, B, T, HW
        for q in range(P):
            g.f0[q] = group.f0[q]
            g.dst[q] = group.ranks[q].bufs[name][0].data_ptr()
        g.f0[P] = T
        self.g = g

    def attach(self, d):
        d.peer = C.addressof(self.g)
        d.out, d.ldo = self.own.data_ptr(), self.C

    def finish(self, part):
        return part


def scatter_case_ok(P: int, T: int, B: int, HW: int, Cc: int) -> bool:
    """The product's fused-scatter predicate for a group of P ranks, with the per-group rank limit raised to the 4 ranks the kernel
    supports (VC_PEER_FUSED_MAXP=4) and the default 'aligned' shape set."""
    return parallel.fused_scatter_ok("aligned", 4, 4, parallel.frame_ranges(T, P), B, HW, Cc)


# -- layout definitions (FrameComm._to_sites / _to_frames): X is the full [B, T, HW, C] tensor -----------------------------------------
def frames_of(X: torch.Tensor, ranges, r: int) -> torch.Tensor:
    """Rank r's frame-layout rows [(b, t_local, hw), C]."""
    f0, f1 = ranges[r]
    return X[:, f0:f1].reshape(-1, X.shape[3]).contiguous()


def sites_of(X: torch.Tensor, P: int, q: int) -> torch.Tensor:
    """Rank q's site-layout rows [(b, t, hw_local), C]."""
    HWl = X.shape[2] // P
    return X[:, :, q * HWl:(q + 1) * HWl].reshape(-1, X.shape[3]).contiguous()


def from_frames(parts, ranges, B: int, HW: int) -> torch.Tensor:
    """Inverse of frames_of: every rank's frame-layout rows -> [B, T, HW, C]."""
    return torch.cat([p.view(B, f1 - f0, HW, -1) for p, (f0, f1) in zip(parts, ranges)], 1)


def from_sites(parts, B: int, T: int) -> torch.Tensor:
    """Inverse of sites_of: every rank's site-layout rows -> [B, T, HW, C]."""
    return torch.cat([p.view(B, T, -1, p.shape[1]) for p in parts], 2)


def group_sums(x: torch.Tensor, B: int) -> torch.Tensor:
    """float64 [B, 32, 2] (sum, sumsq) per (sample, group) of rows [B * n, C], and the float64 [B, 32, 2] sums of |x| and x^2."""
    xd = x.double().view(B, -1, 32, x.shape[1] // 32)
    s = torch.stack([xd.sum(dim=(1, 3)), xd.square().sum(dim=(1, 3))], -1)
    a = torch.stack([xd.abs().sum(dim=(1, 3)), xd.square().sum(dim=(1, 3))], -1)
    return s, a



# -- fp32 summation bound ---------------------------------------------------------------------------------------------------------------
# A sum computed in fp32 by any tree whose longest leaf-to-root path has `depth` additions is within depth u / (1 - depth u) * sum |x_i|
# of the exact sum (u = 2^-24; each fp16 square is exact in fp32, so the same holds for the sum of squares with x_i^2).
U = 2.0 ** -24


def depth_exchange(rows_local: int, Cc: int) -> int:
    """peer_exchange_kernel: a thread adds its rows of a split in order (at most ceil(rows_local / ppi)), the CTA adds ppi * cg thread
    sums in order, the last CTA adds the splits (at most 512).  Holds for every grid size."""
    ppi = max(1, 512 // (Cc // 8))
    return -(-rows_local // ppi) + ppi * (Cc // 32) + 512


def depth_records(rows_per_sample: int, Cc: int) -> int:
    """A GEMM's GroupNorm records (gn_part) through groupnorm_parts_to_partials and gn_peer_allreduce_kernel: at most 32 values of a
    row per piece, a 5-level warp reduction per 32-row block, a thread's blocks in order (at most all of them), up to 256 lanes, two
    pieces per sub-group of the group, up to 64 splits."""
    return 32 + 5 + -(-rows_per_sample // 32) + 256 + 2 * (Cc // 32) + 64


def sums_ratio(got: torch.Tensor, ref: torch.Tensor, abss: torch.Tensor, depth: int) -> float:
    """max |got - ref| / bound over every (sum, sumsq); raises AssertionError when a value is outside its bound or not finite."""
    g = depth * U / (1.0 - depth * U)
    bound = g * abss + 1e-30
    got = got.double()
    assert bool(torch.isfinite(got).all()), "non-finite statistics"
    ratio = float(((got - ref).abs() / bound).max())
    assert ratio <= 1.0, f"statistics outside the fp32 summation bound (worst error / bound {ratio:.3g}, depth {depth})"
    return ratio
