"""Frame-sharded multi-GPU execution of the U-Net forward (one process per GPU, torch.distributed / NCCL over NVLink).

SURVEY.md 8(e): every spatial op (2-D convs, per-frame GroupNorm, SpatialTransformer incl. attention, Down/Upsample)
is independent per frame, so rank r owns a contiguous range of the T frames.  The ops that couple frames --
TemporalTransformer (17 per forward) and TemporalConvBlock (22 per forward), including their 5-D GroupNorm statistics
-- run in the transposed "site" layout: every rank holds ALL T frames of H*W/P pixels (H*W is divisible by 8 at every
level), which is perfectly balanced.  The two layouts are exchanged with ONE uneven all-to-all each way
(NCCL all_to_all_single over NVSwitch; volume per rank = activation_bytes * (P-1)/P^2) and the 5-D GroupNorm adds a
[B,32,2] all-reduce.  The reference has no multi-GPU path for this (SURVEY.md 2a); this is new functionality.
"""
from __future__ import annotations

import os
from typing import List

import torch

from . import _lib, ops
from .distributions import posterior_class


def frame_ranges(T: int, world: int) -> List[tuple]:
    """Contiguous, as-even-as-possible split of T frames: 25 over 8 -> 4,3,3,3,3,3,3,3."""
    base, extra = divmod(T, world)
    out, f = [], 0
    for r in range(world):
        n = base + (1 if r < extra else 0)
        out.append((f, f + n))
        f += n
    return out


class FrameComm:
    identity_switches = False       # True: to_sites / to_frames return their argument, with the GroupNorm sums its producer left on it

    def __init__(self, dist, rank: int, world: int, group=None):
        self.dist, self.rank, self.world, self.group = dist, rank, world, group
        self.T = None
        self.ranges = None
        self.bytes_moved = 0            # all-to-all payload sent by this rank (for the bench report)
        self._prof = None               # list of (start, end) CUDA events around every exchange when profiling (bench.py: exposed comm time)

    def __bool__(self):
        return self.world > 1

    def bind(self, T: int):
        self.T = T
        self.ranges = frame_ranges(T, self.world)
        return self.ranges[self.rank]

    # -- exposed-communication profile: the exchanges run in-stream, so their device time (incl. waiting for the peers) is exposed --
    def profile(self, on: bool):
        self._prof = [] if on else None

    def profile_ms(self) -> float:
        torch.cuda.synchronize()
        return float(sum(a.elapsed_time(b) for a, b in (self._prof or [])))

    def _mark(self):
        if self._prof is None:
            return None
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def _done(self, e0):
        if e0 is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            self._prof.append((e0, e1))

    # -- layout transposes -----------------------------------------------------------------------
    def to_sites(self, h: torch.Tensor, B: int, HW: int) -> torch.Tensor:
        e0 = self._mark()
        out = self._to_sites(h, B, HW)
        self._done(e0)
        return out

    def to_frames(self, t: torch.Tensor, B: int, HW: int) -> torch.Tensor:
        e0 = self._mark()
        out = self._to_frames(t, B, HW)
        self._done(e0)
        return out

    def _to_sites(self, h: torch.Tensor, B: int, HW: int) -> torch.Tensor:
        """[(b, t_local, hw), C] -> [(b, t_all, hw_local), C]."""
        P, C = self.world, h.shape[1]
        assert HW % P == 0, f"H*W={HW} must be divisible by the world size {P}"
        HWl = HW // P
        Tl = self.ranges[self.rank][1] - self.ranges[self.rank][0]
        send = h.view(B, Tl, P, HWl, C).permute(2, 0, 1, 3, 4).contiguous().view(P * B * Tl * HWl, C)
        out_rows = [B * (f1 - f0) * HWl for f0, f1 in self.ranges]
        recv = torch.empty((sum(out_rows), C), device=h.device, dtype=h.dtype)
        self.dist.all_to_all_single(recv, send, output_split_sizes=out_rows, input_split_sizes=[B * Tl * HWl] * P, group=self.group)
        self.bytes_moved += send.numel() * send.element_size() * (P - 1) // P
        if B == 1:
            return recv                                                   # chunks arrive in frame order already
        parts = [c.view(B, -1, HWl, C) for c in torch.split(recv, out_rows, 0)]
        return torch.cat(parts, dim=1).reshape(B * self.T * HWl, C)

    def _to_frames(self, t: torch.Tensor, B: int, HW: int) -> torch.Tensor:
        """[(b, t_all, hw_local), C] -> [(b, t_local, hw), C]."""
        P, C = self.world, t.shape[1]
        HWl = HW // P
        Tl = self.ranges[self.rank][1] - self.ranges[self.rank][0]
        in_rows = [B * (f1 - f0) * HWl for f0, f1 in self.ranges]
        if B == 1:
            send = t
        else:
            t4 = t.view(B, self.T, HWl, C)
            send = torch.cat([t4[:, f0:f1].reshape(-1, C) for f0, f1 in self.ranges], 0)
        recv = torch.empty((P * B * Tl * HWl, C), device=t.device, dtype=t.dtype)
        self.dist.all_to_all_single(recv, send.contiguous(), output_split_sizes=[B * Tl * HWl] * P, input_split_sizes=in_rows, group=self.group)
        self.bytes_moved += (send.numel() - in_rows[self.rank] * C) * send.element_size()
        return recv.view(P, B, Tl, HWl, C).permute(1, 2, 0, 3, 4).contiguous().view(B * Tl * HW, C)

    def all_reduce(self, t: torch.Tensor):
        self.dist.all_reduce(t, group=self.group)

    def scatter_plan(self, to_sites: bool, B: int, HW: int, Cc: int):
        """No fused switch with NCCL collectives (see PeerFrameComm.scatter_plan): the caller switches separately."""
        return None

    def owns(self, t: torch.Tensor) -> bool:
        return False

    def groupnorm5d(self, x, B, gamma, beta, eps, silu, stat_rows, fresh: bool):
        """GroupNorm(32) of a site-layout tensor whose statistics span the ranks of the group.  `fresh`: x is the tensor the
        last to_sites() returned (the peer-memory path already holds its statistics)."""
        if ops.reproducible():
            return self._groupnorm5d_leaves(x, B, gamma, beta, eps, silu, stat_rows)
        st = ops.groupnorm_stats(x, B)
        e0 = self._mark()
        self.all_reduce(st)
        self._done(e0)
        return ops.groupnorm_apply(x, B, st, stat_rows, gamma, beta, eps, silu)

    # -- reproducible mode: canonical GroupNorm leaves (ops.groupnorm_canonical) ------------------------------------------------
    def leaf_geometry(self, stat_rows: int):
        """(HW, nc, rows per leaf) of a site-layout 5-D GroupNorm over stat_rows = T * HW rows per sample: this rank holds the chunks
        [rank * nc / P, (rank + 1) * nc / P) of every frame, whole, so its leaves are exactly those of a single GPU."""
        HW = stat_rows // self.T
        nc = ops.gn_leaf_chunks(HW)
        if nc % self.world != 0:
            raise ValueError(f"reproducible mode: a frame group of {self.world} GPUs does not divide the {nc} GroupNorm chunks of "
                             f"{HW}-pixel frames (frame groups of 2, 4 or 8 GPUs need H*W divisible by 8)")
        return HW, nc, HW // nc

    def gather_leaves(self, leaves: torch.Tensor, B: int, nc: int) -> torch.Tensor:
        """This rank's leaves [(b, t, chunk_local), 32, 2] -> every rank's, in canonical [(b, t, chunk), 32, 2] order (exact copies)."""
        P = self.world
        ncl = nc // P
        parts = leaves.new_empty((P,) + tuple(leaves.shape))
        e0 = self._mark()
        self.dist.all_gather_into_tensor(parts.view(-1), leaves.contiguous().view(-1), group=self.group)
        self._done(e0)
        return parts.view(P, B * self.T, ncl, 64).permute(1, 0, 2, 3).reshape(B * self.T * nc, 32, 2).contiguous()

    def _groupnorm5d_leaves(self, x, B, gamma, beta, eps, silu, stat_rows):
        HW, nc, rows_per_leaf = self.leaf_geometry(stat_rows)
        leaves = self.gather_leaves(ops.groupnorm_leaves(x, rows_per_leaf), B, nc)
        return ops.groupnorm_apply_leaves(x, B, leaves, stat_rows, gamma, beta, eps, silu)

    def gather_frames(self, y_local: torch.Tensor, T: int) -> torch.Tensor:
        """[B,C,T_local,H,W] per rank -> the full [B,C,T,H,W] on every rank (3.7 MB at the headline size)."""
        B, C, _, H, W = y_local.shape
        tmax = max(f1 - f0 for f0, f1 in self.ranges)
        mine = y_local.new_zeros((B, C, tmax, H, W))
        mine[:, :, :y_local.shape[2]] = y_local
        parts = y_local.new_empty((self.world, B, C, tmax, H, W))
        self.dist.all_gather_into_tensor(parts.view(-1), mine.view(-1), group=self.group)       # uneven frame counts: padded to the largest shard
        return torch.cat([parts[r, :, :, :f1 - f0] for r, (f0, f1) in enumerate(self.ranges)], dim=2)


class LocalFrameComm(FrameComm):
    """The frame group of one GPU, which UNetModel runs through when it is not frame-sharded over several: it owns all T frames, its
    layout switches and frame gather return their argument, and its 5-D GroupNorm takes its statistics locally.  Opens no process group."""
    identity_switches = True

    def __init__(self):
        super().__init__(None, 0, 1)

    def to_sites(self, h: torch.Tensor, *_) -> torch.Tensor:
        return h
    to_frames = gather_frames = to_sites

    def groupnorm5d(self, x, B, gamma, beta, eps, silu, stat_rows, fresh: bool):
        if ops.reproducible():
            return ops.groupnorm_canonical(x, B, stat_rows // self.T, gamma, beta, eps, silu)
        return ops.groupnorm(x, B, gamma, beta, eps, silu)


class PeerFrameComm(FrameComm):
    """FrameComm whose layout switches and GroupNorm statistics run as this library's own kernels over NVLink peer memory
    (csrc/peer.cu) instead of NCCL collectives: every rank maps the receive buffers, flag words and statistics slots of the
    other ranks of its group (CUDA IPC: cudaMalloc'd buffers, handles exchanged once over the process group, opened with the
    importing rank's compute device current) and
      * to_sites / to_frames are ONE kernel each (rows stored straight into the owning rank's buffer; no pack / unpack copy),
      * the statistics of the 5-D GroupNorm that follows every to_sites ride along with it (no statistics pass, no all-reduce),
      * the GroupNorms in the middle of a temporal block exchange 2 x 32 floats per sample through the same flag protocol.
    The receive buffers are reused by every switch (one per direction): tensors returned by to_sites()/to_frames() are views
    of them and are only valid until the next switch in the same direction -- UNetModel clones the ones it keeps as skips.
    Batches of up to `bmax` samples (4: the B=3 forward of three-way guidance); the receive buffers grow with the first
    switch that needs more room."""

    def __init__(self, dist, rank: int, world: int, group, device, bmax: int = 4):
        super().__init__(dist, rank, world, group)
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.bmax = bmax
        self._bufs = {}            # name -> (own tensor, [device pointer of rank q's buffer as mapped here], capacity in elements)
        self._leaves = None        # the same for the GroupNorm leaves of reproducible mode (float32, two halves of `capacity`)
        self._own_ptrs, self._peer_ptrs = [], []
        with torch.cuda.device(self.device):
            self.seq = torch.zeros(1, dtype=torch.int32, device=self.device)
            self.done = torch.zeros(1, dtype=torch.int32, device=self.device)
            self.cur_stats = torch.zeros((bmax, world, 32, 2), dtype=torch.float32, device=self.device)
            self.ws = torch.empty(bmax * 512 * 64, dtype=torch.float32, device=self.device)
            torch.cuda.synchronize()
            self.flags, flag_ptrs = self._shared(world * 4, torch.int32)
            self.slots, slot_ptrs = self._shared(2 * bmax * world * 64 * 4, torch.float32)
        c = _lib.PeerComm()
        c.world, c.rank, c.Bmax = world, rank, bmax
        c.flags, c.seq, c.done, c.cur_stats = self.flags.data_ptr(), self.seq.data_ptr(), self.done.data_ptr(), self.cur_stats.data_ptr()
        for q in range(world):
            c.peer_flags[q] = flag_ptrs[q]
            c.stats_slots[q] = slot_ptrs[q]
        self.c = c
        self._stats_of = None      # data_ptr of the tensor whose statistics cur_stats holds
        # layout switches inside the producing GEMM's epilogue (scatter_plan): "0" off, "1" every supported shape, "aligned" (default) only
        # shapes whose 32-row epilogue patches never straddle a rank's pixel range or a frame (H*W/P and H*W multiples of 32)
        self.fused = os.environ.get("VC_PEER_FUSED", "aligned")
        # ... and only for frame groups of at most this many ranks: 2 is the largest group the fused switches were checked with on
        # multi-GPU hardware (probe at the real level shapes, sharded forward vs single GPU, graph replay); the kernels handle up to 4
        # ranks (VC_PEER_FUSED_MAXP=4)
        self.fused_max_p = int(os.environ.get("VC_PEER_FUSED_MAXP", "2"))
        self.fused_switches = 0

    # -- CUDA IPC plumbing (setup only) -------------------------------------------------------------
    class _Raw:
        """__cuda_array_interface__ over a raw device allocation, so torch can alias it."""

        def __init__(self, ptr, nbytes):
            self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}

    def _shared(self, nbytes: int, dtype):
        """A zero-filled IPC-shareable allocation of `nbytes` on EVERY rank of the group (collective).  Returns (own tensor of
        `dtype`, [device pointer of rank q's allocation as mapped into this process]); the mapping is opened with this rank's
        compute device current, which is what gives its kernels access over NVLink."""
        import ctypes as C
        nbytes = (int(nbytes) + 255) // 256 * 256
        ptr, handle = C.c_void_p(), (C.c_uint8 * 64)()
        _lib.check(self.lib.vc_peer_alloc(nbytes, C.byref(ptr), handle), "vc_peer_alloc")
        self._own_ptrs.append(ptr.value)
        handles = [None] * self.world
        self.dist.all_gather_object(handles, (bytes(handle), torch.cuda.current_device()), group=self.group)
        ptrs = []
        for q, (hb, dev_q) in enumerate(handles):
            if q == self.rank:
                ptrs.append(ptr.value)
                continue
            _lib.check(self.lib.vc_enable_peer_access(int(dev_q)), "vc_enable_peer_access")
            rp = C.c_void_p()
            _lib.check(self.lib.vc_peer_open((C.c_uint8 * 64).from_buffer_copy(hb), C.byref(rp)), "vc_peer_open")
            self._peer_ptrs.append(rp.value)
            ptrs.append(rp.value)
        own = torch.as_tensor(self._Raw(ptr.value, nbytes), device=self.device).view(dtype)
        self.dist.barrier(group=self.group)
        return own, ptrs

    def _buffer(self, name: str, numel: int):
        """fp16 receive buffer `name` with room for `numel` elements on EVERY rank (collective: all ranks grow it together)."""
        ent = self._bufs.get(name)
        if ent is None or ent[2] < numel:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("PeerFrameComm: a receive buffer must grow during CUDA-graph capture; run one eager forward first")
            torch.cuda.synchronize()
            self.dist.barrier(group=self.group)          # nobody still writes into the old mapping
            with torch.cuda.device(self.device):
                own, ptrs = self._shared(numel * 2, torch.float16)
            ent = (own, ptrs, numel)
            self._bufs[name] = ent
        return ent

    def _exchange(self, h: torch.Tensor, B: int, HW: int, to_sites: bool) -> torch.Tensor:
        import ctypes as C
        P, Cc = self.world, h.shape[1]
        assert HW % P == 0, f"H*W={HW} must be divisible by the world size {P}"
        assert h.is_contiguous() and h.dtype == torch.float16 and B <= self.bmax
        HWl = HW // P
        Tl = self.ranges[self.rank][1] - self.ranges[self.rank][0]
        tmax = max(f1 - f0 for f0, f1 in self.ranges)
        out_rows = B * self.T * HWl if to_sites else B * Tl * HW
        cap = B * (self.T * HWl if to_sites else tmax * HW) * Cc        # same on every rank
        own, ptrs, _ = self._buffer("sites" if to_sites else "frames", cap)
        dst = (C.c_void_p * P)(*ptrs)
        f0 = (C.c_int32 * (P + 1))(*([r[0] for r in self.ranges] + [self.T]))
        with_stats = to_sites and not ops.reproducible()          # reproducible mode takes its statistics from leaves
        _lib.check(self.lib.vc_peer_exchange(C.byref(self.c), h.data_ptr(), dst, int(to_sites), B, self.T, HW, Cc, f0, int(with_stats),
                                             self.ws.data_ptr(), self.ws.numel() * 4, torch.cuda.current_stream().cuda_stream), "vc_peer_exchange")
        sent = h.numel() * 2
        self.bytes_moved += sent * (P - 1) // P if to_sites else sent - B * Tl * HWl * Cc * 2
        out = own[:out_rows * Cc].view(out_rows, Cc)
        self._stats_of = out.data_ptr() if with_stats else None
        return out

    def _to_sites(self, h: torch.Tensor, B: int, HW: int) -> torch.Tensor:
        return self._exchange(h, B, HW, True)

    def _to_frames(self, t: torch.Tensor, B: int, HW: int) -> torch.Tensor:
        return self._exchange(t, B, HW, False)

    def gather_leaves(self, leaves: torch.Tensor, B: int, nc: int) -> torch.Tensor:
        """FrameComm.gather_leaves through peer memory: one kernel stores this rank's leaves into their canonical place of every rank's
        leaf buffer and, after the rendezvous, copies the gathered array out (graph-capturable, no NCCL call)."""
        import ctypes as C
        n = B * self.T * nc * 64
        own, ptrs, cap = self._leaf_buffer(n)
        out = torch.empty((B * self.T * nc, 32, 2), device=leaves.device, dtype=torch.float32)
        e0 = self._mark()
        _lib.check(self.lib.vc_peer_gather_leaves(C.byref(self.c), leaves.contiguous().data_ptr(), (C.c_void_p * self.world)(*ptrs), cap, B,
                                                  self.T, nc, out.data_ptr(), torch.cuda.current_stream().cuda_stream), "vc_peer_gather_leaves")
        self._done(e0)
        return out

    def _leaf_buffer(self, numel: int):
        """float32 [2][cap] leaf buffer on every rank (collective growth, like _buffer) -> (own, peer pointers, cap)."""
        ent = self._leaves
        if ent is None or ent[2] < numel:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("PeerFrameComm: the leaf buffer must grow during CUDA-graph capture; run one eager forward first")
            torch.cuda.synchronize()
            self.dist.barrier(group=self.group)
            with torch.cuda.device(self.device):
                own, ptrs = self._shared(2 * numel * 4, torch.float32)
            ent = (own, ptrs, numel)
            self._leaves = ent
        return ent

    def groupnorm5d(self, x, B, gamma, beta, eps, silu, stat_rows, fresh: bool):
        import ctypes as C
        if ops.reproducible():
            self._stats_of = None
            return self._groupnorm5d_leaves(x, B, gamma, beta, eps, silu, stat_rows)
        stream = torch.cuda.current_stream().cuda_stream
        rows, Cc = x.shape
        if not (fresh and self._stats_of == x.data_ptr()):
            e0 = self._mark()
            _lib.check(self.lib.vc_peer_groupnorm_stats(C.byref(self.c), x.data_ptr(), Cc, B, rows // B, self.ws.data_ptr(), self.ws.numel() * 4,
                                                        stream), "vc_peer_groupnorm_stats")
            self._done(e0)
        self._stats_of = None
        out = torch.empty_like(x)
        _lib.check(self.lib.vc_groupnorm_apply_parts(x.data_ptr(), Cc, B, rows // B, self.cur_stats.data_ptr(), self.world, stat_rows,
                                                     gamma.data_ptr(), beta.data_ptr(), eps, int(silu), out.data_ptr(), stream),
                   "vc_groupnorm_apply_parts")
        return out

    # -- layout switch fused into the producing GEMM's epilogue ------------------------------------------------
    def scatter_plan(self, to_sites: bool, B: int, HW: int, Cc: int):
        """A plan for ops.conv3x3 / conv_temporal / linear(peer=plan): the GEMM that PRODUCES the tensor stores its output tiles straight
        into the receive buffers of the ranks that own them in the other layout (TMA stores over NVLink, overlapped with its MMAs), and
        a one-CTA kernel completes the switch (rendezvous + the cross-rank GroupNorm sums from the GEMM's own partial sums).  Replaces
        GEMM -> local tensor -> peer_exchange_kernel.  None when the shape is not supported (the caller then switches separately)."""
        if not fused_scatter_ok(self.fused, self.fused_max_p, self.bmax, self.ranges, B, HW, Cc):
            return None
        return _ScatterPlan(self, to_sites, B, HW, Cc)

    def owns(self, t: torch.Tensor) -> bool:
        """True if `t` is a view of one of the reusable receive buffers."""
        p = t.data_ptr()
        return any(ent[0].data_ptr() <= p < ent[0].data_ptr() + ent[0].numel() * 2 for ent in self._bufs.values())

    def close(self):
        """Unmap the peers' buffers and free the own ones (call on every rank after a barrier; optional at process exit)."""
        for p in self._peer_ptrs:
            self.lib.vc_peer_close(p)
        for p in self._own_ptrs:
            self.lib.vc_peer_free(p)
        self._peer_ptrs, self._own_ptrs, self._bufs, self._leaves = [], [], {}, None


def fused_scatter_ok(fused: str, fused_max_p: int, bmax: int, ranges, B: int, HW: int, Cc: int) -> bool:
    """Whether a layout switch of B samples of HW pixels and Cc channels over a frame group with the frame ranges `ranges` (one per
    rank) may run in the producing GEMM's epilogue (PeerFrameComm.scatter_plan).  `fused`, `fused_max_p`: PeerFrameComm's settings
    (VC_PEER_FUSED, VC_PEER_FUSED_MAXP); bmax: the largest batch of the group's buffers."""
    P = len(ranges)
    if fused == "0" or P > min(4, fused_max_p) or HW % P != 0 or Cc % 32 != 0 or B > bmax:
        return False
    if fused == "aligned" and ((HW // P) % 32 != 0 or HW % 32 != 0):
        return False
    # the decision must be the same on every rank of the group: it depends on ALL frame ranges, not on this rank's
    for f0, f1 in ranges:
        if f1 - f0 == 0 or (B > 1 and ((f1 - f0) * HW) % 128 != 0):
            return False
    return True


class _ScatterPlan:
    """One fused layout switch (PeerFrameComm.scatter_plan): attach() fills the GEMM descriptor, finish() completes the switch."""

    def __init__(self, comm: "PeerFrameComm", to_sites: bool, B: int, HW: int, Cc: int):
        self.comm, self.to_sites, self.B, self.HW, self.C = comm, to_sites, B, HW, Cc
        P = comm.world
        HWl = HW // P
        Tl = comm.ranges[comm.rank][1] - comm.ranges[comm.rank][0]
        tmax = max(f1 - f0 for f0, f1 in comm.ranges)
        self.rows_in = B * Tl * HW if to_sites else B * comm.T * HWl
        self.rows_out = B * comm.T * HWl if to_sites else B * Tl * HW
        cap = B * (comm.T * HWl if to_sites else tmax * HW) * Cc            # same on every rank (as in _exchange)
        self.own, ptrs, _ = comm._buffer("sites" if to_sites else "frames", cap)
        g = _lib.GemmPeer()
        g.mode, g.world, g.rank, g.B, g.T, g.HW = (1 if to_sites else 2), P, comm.rank, B, comm.T, HW
        for q in range(P):
            g.f0[q] = comm.ranges[q][0]
            g.dst[q] = ptrs[q]
        g.f0[P] = comm.T
        self.g = g

    def attach(self, d):
        """Route the output of the GEMM described by `d` (its `out` must not be set by the caller)."""
        import ctypes as C
        d.peer = C.addressof(self.g)
        d.out, d.ldo = self.own.data_ptr(), self.C            # never written: the epilogue stores through the per-rank maps

    def finish(self, gn_part):
        """Rendezvous (+ cross-rank GroupNorm sums for frames -> sites).  Returns the switched tensor (a view of the receive buffer)."""
        import ctypes as C
        comm = self.comm
        geom = None
        if self.to_sites and gn_part is not None:
            Tl = comm.ranges[comm.rank][1] - comm.ranges[comm.rank][0]
            geom = gn_part.geom(self.B, Tl * self.HW)
        # geom None (channel counts whose GroupNorm groups are not multiples of the 10-channel sub-groups, e.g. reduced test widths):
        # rendezvous only; groupnorm5d() then takes its statistics with a pass over the received tensor (vc_peer_groupnorm_stats)
        e0 = comm._mark()
        _lib.check(comm.lib.vc_peer_finish_scatter(C.byref(comm.c), C.byref(geom) if geom is not None else None, self.C, self.B, comm.ws.data_ptr(),
                                                   comm.ws.numel() * 4, torch.cuda.current_stream().cuda_stream), "vc_peer_finish_scatter")
        comm._done(e0)
        P = comm.world
        sent = self.rows_in * self.C * 2
        Tl = comm.ranges[comm.rank][1] - comm.ranges[comm.rank][0]
        comm.bytes_moved += sent * (P - 1) // P if self.to_sites else sent - self.B * Tl * (self.HW // P) * self.C * 2
        comm.fused_switches += 1
        out = self.own[:self.rows_out * self.C].view(self.rows_out, self.C)
        comm._stats_of = out.data_ptr() if geom is not None else None
        return out


class CfgComm:
    """Classifier-free-guidance split: the conditional and unconditional U-Net forwards of a DDIM step are independent
    (ddim.py:223-224), so the first half of the ranks computes `cond`, the second half `uncond`, and rank i swaps its
    3.7 MB prediction with rank i + world/2 through a 2-rank all-gather.  Three-way guidance (ddim_multiplecond.py) puts
    `uncond` and `uncond_img` on the second half, which then sends twice the rows of the first."""

    def __init__(self, dist, branch: int, pair_group):
        self.dist, self.branch, self.pair_group = dist, branch, pair_group

    def exchange(self, v_mine: torch.Tensor, rows=None):
        """-> (branch 0's prediction, branch 1's prediction).  `rows`: the batch rows of the two when they differ; the smaller
        part is zero-padded to the larger for the all-gather."""
        rows = rows or (v_mine.shape[0], v_mine.shape[0])
        n = max(rows)
        mine = v_mine.contiguous()
        if mine.shape[0] < n:
            mine = torch.cat([mine, mine.new_zeros((n - mine.shape[0], *mine.shape[1:]))], 0)
        buf = v_mine.new_empty((2, n, *v_mine.shape[1:]))
        self.dist.all_gather_into_tensor(buf.view(-1), mine.view(-1), group=self.pair_group)   # pair group rank order = (branch 0, branch 1)
        return buf[0, :rows[0]], buf[1, :rows[1]]


# -- the VAE, frame-sharded over all ranks -----------------------------------------------------------------------------------------
# The VAE is a 2-D network applied to every frame on its own (SURVEY.md 8(e)): frame f of the clip flattened as (b t) depends on
# input frame f only.  Rank r encodes / decodes the frames frame_ranges(B*T, world)[r] and the shares are all-gathered; under the
# CFG split too, since the VAE has no guidance branches.  The *_share functions compute one rank's share without a process group.

def _flat_frames(x: torch.Tensor) -> torch.Tensor:
    """[b, c, t, h, w] -> [(b t), c, h, w], the frame order of encode_first_stage / decode_core (ddpm3d.py:620-667)."""
    b, c, t, h, w = x.shape
    return x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)


def vae_encode_share(model, videos: torch.Tensor, rank: int, world: int):
    """Rank `rank`'s share of encoding videos [b, 3, t, H, W]: the fp32 posterior moments [n_r, 2*embed_dim, H/8, W/8] of its frames,
    one first_stage_model.encode call per frame when model.perframe_ae, else one call for all of them (as encode_first_stage calls
    it).  None for a rank without frames.  Draws no random numbers; vae_latents_from_moments samples the posterior."""
    f0, f1 = frame_ranges(videos.shape[0] * videos.shape[2], world)[rank]
    if f1 == f0:
        return None
    x = _flat_frames(videos)[f0:f1]
    encode = model.first_stage_model.encode
    if model.perframe_ae:
        return torch.cat([encode(x[i:i + 1]).parameters for i in range(f1 - f0)], 0)
    return encode(x).parameters


def vae_latents_from_moments(model, moments: torch.Tensor, b: int, t: int) -> torch.Tensor:
    """The moments of all b*t frames [(b t), 2*embed_dim, h, w] -> latents [b, embed_dim, t, h, w], sampled as encode_first_stage
    samples them: one get_first_stage_encoding per frame when model.perframe_ae, else one over all frames.  The posterior draws
    come from the CPU generator (distributions.py), so every rank replays all frames in order: each then leaves that generator in
    the state a single process leaves it in."""
    post = posterior_class()
    if model.perframe_ae:
        z = torch.cat([model.get_first_stage_encoding(post(moments[i:i + 1])).detach() for i in range(moments.shape[0])], 0)
    else:
        z = model.get_first_stage_encoding(post(moments)).detach()
    return z.reshape(b, t, *z.shape[1:]).permute(0, 2, 1, 3, 4)


def vae_decode_share(model, z: torch.Tensor, rank: int, world: int):
    """Rank `rank`'s share of decode_first_stage(z) for latents z [b, c, t, h, w]: the model's own decode_first_stage on its frames
    as one 4-D [n_r, c, h, w] tensor (so perframe_ae and decode_batch apply as the model defines them) -> [n_r, 3, H, W].
    None for a rank without frames."""
    f0, f1 = frame_ranges(z.shape[0] * z.shape[2], world)[rank]
    if f1 == f0:
        return None
    return model.decode_first_stage(_flat_frames(z)[f0:f1])


def gather_shares(comm: FrameComm, share, n: int, device, dtype) -> torch.Tensor:
    """Every rank's share [n_r, C, H, W] of n frames (None on a rank without frames, which then contributes an empty share of
    `dtype`) -> all n frames [n, C, H, W] on every rank: one all-gather padded to the largest share (FrameComm.gather_frames).
    When n < world the ranks without frames first learn C, H, W from rank 0, which always holds a frame."""
    comm.bind(n)
    if n < comm.world:
        dims = torch.tensor(list(share.shape[1:]) if share is not None else [0, 0, 0], dtype=torch.int64, device=device)
        comm.dist.broadcast(dims, 0, group=comm.group)
        if share is None:
            share = torch.empty((0, *dims.tolist()), device=device, dtype=dtype)
    return comm.gather_frames(share.permute(1, 0, 2, 3).unsqueeze(0), n)[0].transpose(0, 1)


def vae_encode(model, videos: torch.Tensor) -> torch.Tensor:
    """synthesis.get_latent_z sharded over the ranks of model._vae_comm (set by shard_model): videos [b, 3, t, H, W] -> latents
    [b, embed_dim, t, H/8, W/8] on every rank.  The moments are all-gathered (fp32, 7.4 MB at 576x1024x25)."""
    comm = model._vae_comm
    b, t = videos.shape[0], videos.shape[2]
    share = vae_encode_share(model, videos, comm.rank, comm.world)
    moments = gather_shares(comm, share, b * t, videos.device, torch.float32).contiguous()
    return vae_latents_from_moments(model, moments, b, t)


def vae_decode(model, z: torch.Tensor) -> torch.Tensor:
    """model.decode_first_stage(z) sharded over the ranks of model._vae_comm: latents [b, c, t, h, w] -> [b, 3, t, H, W] on every
    rank, in the dtype decode_first_stage returns (the latents' for AutoencoderKL)."""
    comm = model._vae_comm
    b, t = z.shape[0], z.shape[2]
    share = vae_decode_share(model, z, comm.rank, comm.world)
    y = gather_shares(comm, share, b * t, z.device, z.dtype)
    return y.reshape(b, t, *y.shape[1:]).permute(0, 2, 1, 3, 4)


class Replicas:
    """shard_model(replicas=R): the world cut into R groups of world / R consecutive ranks, each running whole outputs of a synthesis
    call.  synthesis.image_guided_synthesis numbers the outputs j = k * B + b (sample k, clip b) and runs job j on group j % R; a group
    runs its jobs in increasing j.  `index` is this rank's group; collectives go over the default group (the whole world)."""

    def __init__(self, dist, index: int, count: int, world: int):
        self.dist, self.index, self.count, self.world = dist, index, count, world
        self.size = world // count

    def jobs(self, n_jobs: int) -> List[int]:
        """The jobs of this rank's group, in the order it runs them (none when n_jobs <= index: the group is idle)."""
        return list(range(self.index, n_jobs, self.count))

    def gather_jobs(self, mine: List[torch.Tensor], n_jobs: int, shape, device) -> torch.Tensor:
        """This group's job results (fp32 [1, *shape] each, in the order of jobs()) -> all n_jobs results [n_jobs, *shape] in job order, on
        every rank: one all-gather over the world, padded to the largest group's job count (idle groups send padding only).  Every rank
        of a group holds the same results; the first rank's are taken."""
        m = -(-n_jobs // self.count)
        send = torch.zeros((m, *shape), device=device, dtype=torch.float32)
        for i, t in enumerate(mine):
            send[i] = t[0]
        parts = send.new_empty((self.world, m, *shape))
        self.dist.all_gather_into_tensor(parts.view(-1), send.view(-1))
        return torch.stack([parts[(j % self.count) * self.size, j // self.count] for j in range(n_jobs)])


def _make_comm(dist, rank, world, group, device, peer: bool):
    if peer and world > 1 and device is not None and torch.device(device).type == "cuda":
        comm, err = None, None
        try:
            comm = PeerFrameComm(dist, rank, world, group, device)
        except Exception as e:                       # e.g. CUDA IPC not permitted in this container
            err = e
        ok = torch.tensor([0.0 if comm is None else 1.0], device=device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)      # all ranks of the group take the same path
        if float(ok) > 0:
            return comm
        import warnings
        warnings.warn(f"viewcrafter_b200.parallel: NVLink peer-memory exchange unavailable ({err!r}); using the NCCL collectives")
    return FrameComm(dist, rank, world, group)


def shard_model(model, dist, rank: int, world: int, cfg_split: bool = True, peer: bool = None, replicas: int = 1):
    """Distribute the denoise step over `world` ranks (weights stay replicated: 2.9 GB fp16 per GPU).

    world even and cfg_split: 2-way CFG split x (world/2)-way frame sharding -- e.g. 8 GPUs = 2 x 4 with frames 7/6/6/6
    (ideal 7.1x) instead of 8-way frames 4/3x7 (ideal 6.25x).  Otherwise pure frame sharding.
    replicas=R: the world is cut into R groups of G = world / R consecutive ranks and the layout above applies inside each group, to
    G ranks; a group of one rank has no communicator and runs the one-GPU path.  The model gets `model._replicas` (Replicas), and
    synthesis.image_guided_synthesis then runs the samples and clips of one call concurrently, one whole output per group at a time.
    A model with a VAE (`first_stage_model`) also gets `model._vae_comm`, a FrameComm over all `world` ranks of the default group:
    synthesis.get_latent_z and image_guided_synthesis then encode and decode the frames sharded over every rank (vae_encode,
    vae_decode).  That adds no process group and no collective here.
    Every rank must call this (it creates process groups collectively).  Returns the U-Net's FrameComm (or None)."""
    unet = model.model.diffusion_model if hasattr(model, "model") else model
    try:
        device = next(unet.parameters()).device
    except StopIteration:
        device = None
    modes = [None] * world
    dist.all_gather_object(modes, (ops.reproducible(), replicas))
    if len(set(m for m, _ in modes)) != 1:
        raise RuntimeError(f"shard_model: the ranks disagree on reproducible mode ({[m for m, _ in modes]}); call "
                           f"viewcrafter_b200.set_reproducible() or set VC_REPRODUCIBLE the same way on every rank")
    if len(set(r for _, r in modes)) != 1:
        raise ValueError(f"shard_model: the ranks disagree on replicas ({[r for _, r in modes]})")
    if not isinstance(replicas, int) or replicas < 1 or world % replicas != 0:
        raise ValueError(f"shard_model: replicas must be a positive integer that divides the world size {world}, got {replicas!r}")
    G = world // replicas                                  # ranks per replica group; the group of this rank starts at rank `off`
    g, off = rank // G, rank // G * G
    split = cfg_split and G % 2 == 0 and hasattr(model, "model")
    P = G // 2 if split else G
    if ops.reproducible() and P not in (1, 2, 4, 8):
        raise ValueError(f"shard_model: reproducible mode supports frame groups of 1, 2, 4 or 8 GPUs (they divide the GroupNorm chunks "
                         f"of every frame); this layout puts {P} GPUs in a frame group")
    if peer is None:           # NVLink peer-memory kernels on CUDA (VC_PEER_COMM=0: NCCL collectives); the CPU double uses gloo
        peer = os.environ.get("VC_PEER_COMM", "1") != "0"
    if getattr(model, "first_stage_model", None) is not None:
        model._vae_comm = FrameComm(dist, rank, world)
    if replicas > 1:
        model._replicas = Replicas(dist, g, replicas, world)
    if split:
        # every rank creates every group's process groups, in the same order (new_group is collective over the default group)
        groups = [([dist.new_group(list(range(o + b * P, o + (b + 1) * P))) for b in range(2)],
                   [dist.new_group([o + i, o + i + P]) for i in range(P)]) for o in range(0, world, G)]
        frame_groups, pair_groups = groups[g]
        branch, r = (rank - off) // P, (rank - off) % P
        model._cfg = CfgComm(dist, branch, pair_groups[r])
        unet._comm = _make_comm(dist, r, P, frame_groups[branch], device, peer) if P > 1 else None
        return unet._comm
    if replicas == 1:
        unet._comm = _make_comm(dist, rank, world, None, device, peer)
    elif G == 1:
        unet._comm = None
    else:
        groups = [dist.new_group(list(range(o, o + G))) for o in range(0, world, G)]
        unet._comm = _make_comm(dist, rank - off, G, groups[g], device, peer)
    return unet._comm
