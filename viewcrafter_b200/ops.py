"""Torch-tensor wrappers over the C ABI (include/vc_b200.h).  PyTorch is only the allocator / stream provider.

Activation convention: channels-last fp16 matrices ``[rows, C]`` where a row is a pixel of a frame
(``rows = frames*H*W`` in (frame, y, x) order) or a token.  Every function raises on failure; nothing here
falls back to a PyTorch implementation.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import _lib
from ._lib import AttnDesc, DdimScalars, GemmDesc, GnPartGeom, check


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def require_cuda(device, who: str):
    """The product has no CPU path: anything not on a CUDA device is an error, not a fallback."""
    if torch.device(device).type != "cuda":
        raise _lib.VcError(f"{who} runs only on a CUDA (sm_90a) device; there is no CPU path")


VcError = _lib.VcError


def _chk16(t: torch.Tensor, name: str):
    if t.dtype != torch.float16 or not t.is_cuda:
        raise _lib.VcError(f"{name}: expected a CUDA fp16 tensor, got {t.dtype} on {t.device}")
    if t.device.index != torch.cuda.current_device():
        # kernels launch on the CURRENT device's stream: a tensor of another GPU would be dereferenced on the wrong device
        raise _lib.VcError(f"{name}: tensor lives on {t.device} but the current CUDA device is {torch.cuda.current_device()}; "
                           f"wrap the call in torch.cuda.device({t.device.index})")


def launch_count() -> int:
    """Kernel launches issued by the library from the host so far (a captured launch counts once, at capture)."""
    return int(_lib.load().vc_launch_count())


def is_device_only(fn) -> bool:
    """True if an nn.Module._apply function only moves tensors (keeps fp16 and fp32 dtypes)."""
    try:
        a, b = fn(torch.empty(1, dtype=torch.float16)), fn(torch.empty(1, dtype=torch.float32))
        return a.dtype == torch.float16 and b.dtype == torch.float32
    except Exception:
        return False


def tree_apply(obj, fn):
    """fn over every tensor of a nested dict / list / tuple (packed kernel operands)."""
    if isinstance(obj, torch.Tensor):
        return fn(obj)
    if isinstance(obj, dict):
        return {k: tree_apply(v, fn) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(tree_apply(v, fn) for v in obj)
    return obj


def tensor_version(t: torch.Tensor):
    """The in-place version counter, or None for inference tensors (torch.inference_mode()), which do not track one --
    callers then skip caching instead of failing."""
    try:
        return t._version
    except RuntimeError:
        return None


# ----------------------------------------------------------------------------------------------------
# weight packing (host side, once per load_state_dict)
# ----------------------------------------------------------------------------------------------------
def pack_conv3x3(w: torch.Tensor, k_pad: int = 0) -> torch.Tensor:
    """[Cout,Cin,3,3] -> fp16 [9*Cout, Cin(+pad)], tap = ky*3+kx (tap shift dx=kx-1, dy=ky-1)."""
    co, ci = w.shape[0], w.shape[1]
    p = w.permute(2, 3, 0, 1).reshape(9 * co, ci)
    if k_pad > ci:
        p = torch.nn.functional.pad(p, (0, k_pad - ci))
    return p.to(torch.float16).contiguous()


def pack_conv_temporal(w: torch.Tensor) -> torch.Tensor:
    """Conv3d weight [Cout,Cin,3,1,1] -> fp16 [3*Cout, Cin], tap = kt."""
    co, ci = w.shape[0], w.shape[1]
    return w.reshape(co, ci, 3).permute(2, 0, 1).reshape(3 * co, ci).to(torch.float16).contiguous()


def pack_linear(w: torch.Tensor) -> torch.Tensor:
    """[N,K] or 1x1 conv [N,K,1(,1)] -> fp16 [N,K]."""
    return w.reshape(w.shape[0], w.shape[1]).to(torch.float16).contiguous()


def _geglu_index(n2: int, device) -> torch.Tensor:
    inner = n2 // 2
    bn = _lib.load().vc_gemm_tile_n(n2, 1)
    half = bn // 2
    idx = []
    for t in range(n2 // bn):
        idx.extend(range(t * half, (t + 1) * half))
        idx.extend(range(inner + t * half, inner + (t + 1) * half))
    return torch.tensor(idx, device=device)


def pack_geglu(w: torch.Tensor, b: torch.Tensor):
    """GEGLU proj [2*inner, C]: interleave value/gate rows per N tile so the epilogue sees both (attention.py:415-422)."""
    idx = _geglu_index(w.shape[0], w.device)
    return w[idx].to(torch.float16).contiguous(), b[idx].float().contiguous()


def fold_layernorm(w: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, bias: Optional[torch.Tensor] = None):
    """Fold ``LayerNorm(gamma, beta)`` into the linear layer that consumes it (attention.py:283-292: norm1/2/3 feed to_q/k/v
    and the GEGLU projection and nothing else):  W (gamma*xhat + beta) + b  =  rstd * (W' x - mean * colsum(W')) + (W beta + b)
    with W' = W * gamma.  Returns (W' fp16 [N,K], colsum fp32 [N] of the ROUNDED W', bias' fp32 [N]); pair with
    ``linear(x_raw, W', bias=bias', ln=(layernorm_stats(x_raw), colsum))``."""
    w32 = w.reshape(w.shape[0], -1).float()
    w16 = (w32 * gamma.float()[None, :]).to(torch.float16).contiguous()
    colsum = w16.float().sum(1).contiguous()
    b2 = w32 @ beta.float()
    if bias is not None:
        b2 = b2 + bias.float()
    return w16, colsum, b2.contiguous()


def pack_geglu_ln(w: torch.Tensor, b: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor):
    """pack_geglu of a projection with the preceding LayerNorm folded in -> (w16, bias, colsum), rows interleaved per N tile."""
    w16, cs, b2 = fold_layernorm(w, gamma, beta, b)
    idx = _geglu_index(w.shape[0], w.device)
    return w16[idx].contiguous(), b2[idx].contiguous(), cs[idx].contiguous()


FP8_MAX = 448.0     # largest finite e4m3 value


class Fp8Weight:
    """A packed GEMM weight in FP8 mode: e4m3 values ``q`` [taps * N, K] (torch.float8_e4m3fn) and per-output-channel fp32 scales
    ``scale`` [N]; the weight the GEMM multiplies is q * scale[n].  Built by pack_fp8; every tap-GEMM wrapper accepts it for ``w``."""
    __slots__ = ("q", "scale")

    def __init__(self, q: torch.Tensor, scale: torch.Tensor):
        self.q, self.scale = q, scale

    @property
    def shape(self):
        return self.q.shape

    def dequant(self) -> torch.Tensor:
        """fp32 [taps * N, K]: the weights the FP8 GEMM multiplies."""
        taps = self.q.shape[0] // self.scale.shape[0]
        return (self.q.float().view(taps, -1, self.q.shape[1]) * self.scale[None, :, None]).view(self.q.shape)


def pack_fp8(w_packed: torch.Tensor, taps: int = 1):
    """Quantise an already packed fp16 GEMM weight [taps * N, K] (rows tap * N + n) to e4m3 per output channel n:
    s_w[n] = max over taps and k of |w[n]| / 448 (1 for an all-zero channel), q_w = e4m3_rn(w / s_w[n]) (clamped to +-448).
    Returns (q_w as torch.float8_e4m3fn, s_w fp32 [N])."""
    rows, K = w_packed.shape
    assert rows % taps == 0
    w = w_packed.detach().float().view(taps, rows // taps, K)
    amax = w.abs().amax(dim=(0, 2))
    s = torch.where(amax > 0, amax / FP8_MAX, torch.ones_like(amax))
    q = (w / s[None, :, None]).clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
    return q.view(rows, K).contiguous(), s.contiguous()


def fp8_colsum(w8: Fp8Weight) -> torch.Tensor:
    """ln_colsum of a LayerNorm-folded FP8 weight: the column sums of the DEQUANTISED weights, which the GEMM multiplies."""
    return w8.dequant().sum(1).contiguous()


def absmax(x: torch.Tensor, x2: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 [1] device scalar max |[x | x2]| over every row: the per-tensor activation scale of the FP8 GEMM (s_a = amax / 448)."""
    _chk16(x, "absmax.x")
    if x2 is not None:
        _chk16(x2, "absmax.x2")
        assert x2.shape[0] == x.shape[0]
    if out is None:
        out = torch.empty(1, device=x.device, dtype=torch.float32)
    check(_lib.load().vc_absmax_f16(x.data_ptr(), x.shape[0], x.shape[1], x.stride(0), _ptr(x2), 0 if x2 is None else x2.shape[1],
                                    0 if x2 is None else x2.stride(0), out.data_ptr(), _stream()), "vc_absmax_f16")
    return out


# ----------------------------------------------------------------------------------------------------
# tensor-core ops
# ----------------------------------------------------------------------------------------------------
def _gemm(desc: GemmDesc):
    check(_lib.load().vc_gemm_tap(C.byref(desc), _stream()), "vc_gemm_tap")


# GroupNorm statistics from the producing GEMM's epilogue (GemmDesc.gn_part): 0 = off (statistics pass inside the GroupNorm kernel),
# 1 = producers with a long reduction only (3x3 / temporal / stride-2 convs: the extra epilogue work hides under the MMAs), 2 = every producer
GN_FROM_PRODUCER = int(os.environ.get("VC_GN_FROM_PRODUCER", "1"))
# ... taken for every GroupNorm with <= 4 samples (the 5-D ones: one sample = a whole batch element, so the fused kernel's statistics and
# normalise phases cannot overlap across samples) and for per-frame GroupNorms of at least this many MB; smaller per-frame tensors are re-read
# from L2 by the one-launch fused kernel.  Measured on an H100 80GB HBM3 at a 400 W power limit (tools/gn_parts_micro.py, per-frame GroupNorm
# over 50 frames, B = 2): producer sums 283 vs 364 us at 295 MB (level 0), 149 vs 194 at 147 MB, 92 vs 125 at 74 MB, 48 vs 53 at 18 MB
# (level 3) -- the producer sums win at every U-Net level, so the threshold sits below the smallest one
GN_PARTS_MIN_MB = float(os.environ.get("VC_GN_PARTS_MIN_MB", "16"))
# Reproducible mode (set_reproducible / VC_REPRODUCIBLE=1): the same seed gives bit-identical results whatever the batching of the CFG
# branches, the number of GPUs the frames are sharded over, per-frame or batched VAE calls and the SM count of the H100.  GroupNorm
# statistics come from canonical leaves (groupnorm_canonical), the DDIM update launches a fixed grid.  Off by default: the default path
# picks its GroupNorm splits and statistics source for speed, which changes the summation order with the layout.
REPRODUCIBLE = os.environ.get("VC_REPRODUCIBLE", "0") == "1"


def set_reproducible(on: bool = True) -> bool:
    """Switch reproducible mode for the whole process; returns the previous setting.  Models that replay CUDA graphs recapture."""
    global REPRODUCIBLE
    prev, REPRODUCIBLE = REPRODUCIBLE, bool(on)
    return prev


def reproducible() -> bool:
    return REPRODUCIBLE


def gn_leaf_chunks(hw: int) -> int:
    """nc: the chunks a frame of `hw` pixels is cut into for the canonical GroupNorm leaves.  A function of hw alone; a multiple of 8
    whenever hw is (so that the site layout of 2, 4 or 8 GPUs holds whole chunks), doubled while a chunk keeps >= 256 pixels and up to
    1024 chunks, so that even one frame of the VAE decoder (576x1024) spreads over the whole GPU.  1 if hw % 8 != 0."""
    if hw % 8 != 0:
        return 1
    nc = 8
    while nc < 1024 and hw % (2 * nc) == 0 and hw // (2 * nc) >= 256:
        nc *= 2
    return nc


GN_SUB = 10          # sub-group width the U-Net producers cut their chunks at: every GroupNorm(32) boundary of 320 / 640 / 1280 channels
                     # and of their skip concats (640 / 960 / 1280 / 1920 / 2560) is a multiple of 10


class GnPart:
    """The (sum, sumsq) records a GEMM left for the GroupNorm that reads its output: [n_rb, C/32, 4, 2] fp32 over 32-row blocks in
    m-tile order.  `rb_per_z` blocks per producer slab (frame for the 3x3 convs, batch element for the temporal convs, everything
    for a linear); `rows_per_z` valid rows per slab; `row_blocks_linear`: block b of a slab holds the rows [32 b, 32 b + 32) of it."""
    __slots__ = ("part", "n_chunks", "sub", "rb_per_z", "rows_per_z", "slabs", "linear")

    def __init__(self, part, n_chunks, sub, rb_per_z, rows_per_z, slabs, linear):
        self.part, self.n_chunks, self.sub, self.rb_per_z, self.rows_per_z, self.slabs, self.linear = part, n_chunks, sub, rb_per_z, rows_per_z, slabs, linear

    def geom(self, samples: int, rows_per_sample: int):
        """ctypes geometry for a consumer with `samples` x `rows_per_sample` rows, or None if its samples do not fall on block boundaries."""
        g = GnPartGeom()
        g.part, g.n_chunks, g.sub = self.part.data_ptr(), self.n_chunks, self.sub
        total = self.slabs * self.rows_per_z
        if samples * rows_per_sample != total:
            return None
        if rows_per_sample % self.rows_per_z == 0:               # a sample = k whole slabs (k = 1: 4-D GroupNorm after a conv; k = T: 5-D)
            k = rows_per_sample // self.rows_per_z
            g.rb_per_z, g.samples_per_z, g.rb_per_sample = k * self.rb_per_z, 1, k * self.rb_per_z
            return g
        if self.linear and self.rows_per_z % rows_per_sample == 0 and rows_per_sample % 32 == 0:   # several samples per slab
            g.rb_per_z, g.samples_per_z, g.rb_per_sample = self.rb_per_z, self.rows_per_z // rows_per_sample, rows_per_sample // 32
            return g
        return None


def _want_gn(gn_out: bool, k_iters: int) -> bool:
    # reproducible mode never reads the producer's sums (their order follows the GEMM's tiling of the whole batch)
    return bool(gn_out) and not REPRODUCIBLE and (GN_FROM_PRODUCER >= 2 or (GN_FROM_PRODUCER == 1 and k_iters >= 12))


def gn_part_of(t):
    return getattr(t, "_vc_gn", None)


gn_from_parts_calls = 0      # GroupNorms that took their statistics from a producer's partial sums (introspection / tests)


def _tap_gemm(who: str, x: torch.Tensor, w, X: int, Y: int, Z: int, bx: int, by: int, taps, x2: Optional[torch.Tensor] = None,
              amax: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, out_f32: bool = False, ldo: Optional[int] = None,
              ldo_y: int = 0, ldo_z: int = 0, bias: Optional[torch.Tensor] = None, bias_z_div: int = 0, res: Optional[torch.Tensor] = None,
              geglu: bool = False, ln=None, ln_out: bool = False, gn_out: bool = False, peer=None):
    """Launch one tap-GEMM: out[row] = sum over taps (dx, dy) of [x|x2][row shifted by (dx, dy) in the (X, Y, Z) grid] @ w_tap.T, then
    the epilogue options of linear().  w: fp16 [len(taps) * N, K] or an Fp8Weight (amax: the absmax of [x|x2], computed here if None).
    out: written with row pitch ldo (default out.stride(0)) and optional Y / Z pitches; allocated [M, N] if None.  Returns what linear()
    returns."""
    _chk16(x, f"{who}.x")
    fp8 = isinstance(w, Fp8Weight)
    if fp8 and peer is not None:
        raise VcError(f"{who}: FP8 weights do not support the multi-GPU peer-scatter epilogue")
    M, K1 = x.shape
    K = w.shape[1]
    N = w.shape[0] // len(taps)
    n_out = N // 2 if geglu else N
    d = GemmDesc()
    d.a, d.lda = x.data_ptr(), x.stride(0)
    if x2 is not None:
        d.a2, d.lda2 = x2.data_ptr(), x2.stride(0)
        assert K1 + x2.shape[1] == K
    else:
        assert K1 == K, (K1, K)
    d.X, d.Y, d.Z, d.bx, d.by = X, Y, Z, bx, by
    d.K, d.K1, d.N, d.num_taps = K, K1, N, len(taps)
    for t, (dx, dy) in enumerate(taps):
        d.tap_dx[t], d.tap_dy[t] = dx, dy
    if fp8:
        if amax is None:
            amax = absmax(x, x2)
        assert w.q.is_cuda and w.q.dtype == torch.float8_e4m3fn
        d.w, d.ldw = w.q.data_ptr(), w.q.stride(0)
        d.fp8, d.w_scale, d.a_amax = 1, w.scale.data_ptr(), amax.data_ptr()
    else:
        _chk16(w, "gemm.w")
        d.w, d.ldw = w.data_ptr(), w.stride(0)      # w may be a column slice of a wider matrix (e.g. K of a fused QK)
    if peer is not None:
        assert out is None and not geglu and not out_f32 and not ln_out and M == peer.rows_in and N == peer.C
        peer.attach(d)                              # the output goes to the peers' receive buffers
    else:
        if out is None:
            out = torch.empty((M, n_out), device=x.device, dtype=torch.float32 if out_f32 else torch.float16)
        if out_f32:
            d.out_f32 = out.data_ptr()
        else:
            d.out = out.data_ptr()
        d.ldo = out.stride(0) if ldo is None else ldo
        d.ldo_y, d.ldo_z = ldo_y, ldo_z
    d.bias, d.bias_z_div = _ptr(bias), bias_z_div
    if res is not None:
        d.res, d.ldr = res.data_ptr(), res.stride(0)
    d.geglu = int(geglu)
    if ln is not None:
        stats, colsum = ln
        assert stats.shape == (M, 2) and stats.dtype == torch.float32 and stats.is_contiguous()
        assert colsum.shape == (N,) and colsum.dtype == torch.float32 and colsum.is_contiguous()
        d.ln_stats, d.ln_colsum = stats.data_ptr(), colsum.data_ptr()
    # GroupNorm records: a frames -> sites switch always leaves them (the cross-rank GroupNorm sums come from them); a local output
    # when its GroupNorm reads them (gn_out) and the reduction is long enough for the extra epilogue work to hide under the MMAs
    if peer is not None:
        want_gn = peer.to_sites and not REPRODUCIBLE
    else:
        want_gn = _want_gn(gn_out, len(taps) * -(-K // 64)) and not out_f32 and out.is_contiguous()
    part = None
    if want_gn and N % 32 == 0 and N % GN_SUB == 0 and not geglu:
        tx, ty = -(-X // bx), -(-Y // by)
        buf = torch.empty((tx * ty * Z * 4, N // 32, 4, 2), device=x.device, dtype=torch.float32)     # one record row per 32-row block
        d.gn_part, d.gn_sub = buf.data_ptr(), GN_SUB
        part = GnPart(buf, N // 32, GN_SUB, tx * ty * 4, X * Y, Z, linear=(by == 1 and bx == 128 and (Y == 1 or X % 128 == 0)))
    ln_parts = None
    if ln_out and n_out % 32 == 0 and not geglu and not out_f32 and out.is_contiguous():
        ln_parts = torch.empty((n_out // 32, M, 2), device=x.device, dtype=torch.float32)
        d.ln_part = ln_parts.data_ptr()
    _gemm(d)
    if peer is not None:
        return peer.finish(part)
    out._vc_gn = part
    if not ln_out:
        return out
    if ln_parts is None:                            # an output the epilogue cannot gather LayerNorm sums for: a statistics pass
        return out, layernorm_stats(out)
    st = torch.empty((M, 2), device=x.device, dtype=torch.float32)
    check(_lib.load().vc_layernorm_stats_from_parts(ln_parts.data_ptr(), M, n_out, 1e-5, st.data_ptr(), _stream()), "vc_layernorm_stats_from_parts")
    return out, st


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, res: Optional[torch.Tensor] = None,
           geglu: bool = False, out: Optional[torch.Tensor] = None, out_f32: bool = False,
           x2: Optional[torch.Tensor] = None, ln=None, ln_out: bool = False, gn_out: bool = False, peer=None):
    """y = [x|x2] @ w.T (+bias) (GEGLU) (+res).  x: [M,K1] fp16 (row pitch = x.stride(0)), w: [N,K] fp16.
    ln = (stats [M,2] fp32 from layernorm_stats(x), colsum [N] fp32): LayerNorm folded into the epilogue (fold_layernorm).
    ln_out: also return the LayerNorm statistics [M,2] (mean, rstd) of y -- y feeds a LayerNorm next (attention.py:283-292); the
    epilogue leaves per-32-column partial sums of the rows it is writing and a tiny kernel finishes them, so y is not re-read.
    gn_out: y feeds a GroupNorm next: leave its partial sums (GnPart, attached to y as ``y._vc_gn``; see groupnorm()).
    peer: a parallel.PeerFrameComm.scatter_plan(): the epilogue stores y into the other ranks' receive buffers (multi-GPU layout switch
    fused into the GEMM); returns the switched tensor.
    w may be an Fp8Weight (FP8 mode): the absmax of [x|x2] is computed first and the GEMM runs e4m3 x e4m3."""
    return _tap_gemm("linear", x, w, x.shape[0], 1, 1, 128, 1, ((0, 0),), x2=x2, out=out, out_f32=out_f32, bias=bias, res=res,
                     geglu=geglu, ln=ln, ln_out=ln_out, gn_out=gn_out, peer=peer)


def _conv_box(H: int, W: int):
    # widths that divide 128 pack 128/W image rows into one 128-pixel tile; every other width falls back to one
    # (partially filled, TMA zero-filled) tile per 128-pixel row segment -- correct for any W, full speed for the
    # shipped widths (8..128 at the U-Net levels, 128..1024 in the VAE)
    if W >= 128 or 128 % W != 0:
        return 128, 1
    return W, 128 // W


_TAPS_3X3 = tuple((t % 3 - 1, t // 3 - 1) for t in range(9))     # tap = ky * 3 + kx (pack_conv3x3)


def conv3x3(x: torch.Tensor, frames: int, H: int, W: int, w9: torch.Tensor, bias: Optional[torch.Tensor] = None,
            res: Optional[torch.Tensor] = None, x2: Optional[torch.Tensor] = None, bias_z_div: int = 0,
            out_f32: bool = False, out: Optional[torch.Tensor] = None, gn_out: bool = False, peer=None) -> torch.Tensor:
    """3x3 / stride 1 / pad 1 convolution on [frames*H*W, Cin] rows; w9 = pack_conv3x3(weight).  gn_out / peer: see linear()."""
    assert x.shape[0] == frames * H * W, (x.shape[0], frames, H, W)
    return _tap_gemm("conv3x3", x, w9, W, H, frames, *_conv_box(H, W), _TAPS_3X3, x2=x2, out=out, out_f32=out_f32, bias=bias,
                     bias_z_div=bias_z_div, res=res, gn_out=gn_out, peer=peer)


def pack_upconv3x3(w: torch.Tensor):
    """Upsample(nearest x2) followed by a 3x3 / pad 1 conv (openaimodel3d.py:80-106) == four 2x2 convolutions on the SMALL image,
    one per output parity (a, b) = (row & 1, col & 1):  out[2i+a, 2j+b] = sum_{r,c in 0..1} Wab[r][c] . x[i + r + a - 1, j + c + b - 1]
    with the 3x3 taps that land on the same source pixel pre-summed (in fp32, then rounded to fp16): rows a=0: {W[0]}, {W[1]+W[2]};
    a=1: {W[0]+W[1]}, {W[2]}; columns alike.  4/9 of the FLOPs, and the 4x larger upsampled tensor is never materialised.
    Returns 4 packed tensors [(4*Cout), Cin] (tap = r*2 + c) for parities (0,0), (0,1), (1,0), (1,1)."""
    w32 = w.detach().float()
    co, ci = w32.shape[0], w32.shape[1]
    rows = {0: [w32[:, :, 0], w32[:, :, 1] + w32[:, :, 2]], 1: [w32[:, :, 0] + w32[:, :, 1], w32[:, :, 2]]}     # [co, ci, kx] each
    packs = []
    for a in (0, 1):
        for b in (0, 1):
            taps = []
            for r in (0, 1):
                wr = rows[a][r]
                cols = [wr[:, :, 0], wr[:, :, 1] + wr[:, :, 2]] if b == 0 else [wr[:, :, 0] + wr[:, :, 1], wr[:, :, 2]]
                taps.extend(cols)
            packs.append(torch.stack(taps, 0).reshape(4 * co, ci).to(torch.float16).contiguous())
    return packs


def upconv3x3(x: torch.Tensor, frames: int, H: int, W: int, packs, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """conv3x3(upsample2x(x)) on [frames*H*W, Cin] rows -> [frames*2H*2W, Cout]; packs = pack_upconv3x3(weight)."""
    assert x.shape[0] == frames * H * W
    N = packs[0].shape[0] // 4
    assert N % 32 == 0, "upconv3x3 writes through the TMA-store epilogue: Cout must be a multiple of 32"
    out = torch.empty((frames * 4 * H * W, N), device=x.device, dtype=torch.float16)
    amax = absmax(x) if isinstance(packs[0], Fp8Weight) else None      # FP8: one activation scale for the four parities
    for a in (0, 1):
        for b in (0, 1):
            taps = tuple((t % 2 + b - 1, t // 2 + a - 1) for t in range(4))
            # rows from pixel (a, b) of the large image on, every second pixel along x and y
            _tap_gemm("upconv3x3", x, packs[a * 2 + b], W, H, frames, *_conv_box(H, W), taps, amax=amax, out=out[a * 2 * W + b:],
                      ldo=2 * N, ldo_y=4 * W * N, ldo_z=4 * W * H * N, bias=bias)
    return out


def conv_temporal(x: torch.Tensor, B: int, T: int, HW: int, w3: torch.Tensor, bias: Optional[torch.Tensor] = None,
                  res: Optional[torch.Tensor] = None, gn_out: bool = False, peer=None) -> torch.Tensor:
    """Conv3d (3,1,1) pad (1,0,0) on [(B T) HW, C] rows: three row-shifted GEMM taps; batches never mix (Z = B).  gn_out: see linear()."""
    assert x.shape[0] == B * T * HW
    return _tap_gemm("conv_temporal", x, w3, T * HW, 1, B, 128, 1, tuple(((t - 1) * HW, 0) for t in range(3)), bias=bias, res=res,
                     gn_out=gn_out, peer=peer)


def flash_attn(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, B: int, Nq: int, Nk: int, heads: int,
               kv_shared: bool = False, scale: float = 0.125, out: Optional[torch.Tensor] = None,
               accumulate: bool = False) -> torch.Tensor:
    """softmax(q k^T scale) v per head (d=64).  q: [B*Nq, >=heads*64] view, k/v: [Bk*Nk, ...] views (Bk=1 if shared)."""
    _chk16(q, "attn.q"); _chk16(k, "attn.k"); _chk16(v, "attn.v")
    if out is None:
        out = torch.empty((B * Nq, heads * 64), device=q.device, dtype=torch.float16)
    d = AttnDesc()
    d.q, d.ldq = q.data_ptr(), q.stride(0)
    d.k, d.ldk = k.data_ptr(), k.stride(0)
    d.v, d.ldv = v.data_ptr(), v.stride(0)
    assert k.stride(0) == v.stride(0)
    d.out, d.ldo = out.data_ptr(), out.stride(0)
    d.B, d.heads, d.Nq, d.Nk = B, heads, Nq, Nk
    d.kv_batch_stride = 0 if kv_shared else Nk * k.stride(0)
    d.scale = scale
    d.accumulate = int(accumulate)
    check(_lib.load().vc_flash_attn_d64(C.byref(d), _stream()), "vc_flash_attn_d64")
    return out


def temporal_attn(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, T: int, sites: int, heads: int,
                  scale: float = 0.125, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _chk16(q, "tattn.q")
    if out is None:
        out = torch.empty((T * sites, heads * 64), device=q.device, dtype=torch.float16)
    assert out.shape == (T * sites, heads * 64) and out.dtype == torch.float16 and out.stride(1) == 1
    assert q.stride(0) == k.stride(0) == v.stride(0)
    check(_lib.load().vc_temporal_attn(q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), out.data_ptr(), out.stride(0),
                                       T, sites, heads, scale, _stream()), "vc_temporal_attn")
    return out


def temporal_attn_windowed(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, T: int, sites: int, heads: int, W: int, S: int,
                           scale: float = 0.125, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """temporal_attn on overlapping windows of W frames with stride S, blended per frame with the weights min(j + 1, W - j)
    (vc_temporal_attn_windowed; INTEGRATION.md "Long clips: windowed temporal attention").  T <= W is temporal_attn exactly."""
    _chk16(q, "tattn_win.q")
    if out is None:
        out = torch.empty((T * sites, heads * 64), device=q.device, dtype=torch.float16)
    assert out.shape == (T * sites, heads * 64) and out.dtype == torch.float16 and out.stride(1) == 1
    assert q.stride(0) == k.stride(0) == v.stride(0)
    check(_lib.load().vc_temporal_attn_windowed(q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), out.data_ptr(), out.stride(0),
                                                T, sites, heads, W, S, scale, _stream()), "vc_temporal_attn_windowed")
    return out


# ----------------------------------------------------------------------------------------------------
# normalisation / data movement
# ----------------------------------------------------------------------------------------------------
_gn_ws = {}


def _gn_workspace(device, samples: int) -> torch.Tensor:
    need = _lib.load().vc_groupnorm_ws_bytes(samples)
    key = (device, torch.cuda.current_stream().cuda_stream)
    ws = _gn_ws.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(max(need, 1 << 20), device=device, dtype=torch.uint8)
        _gn_ws[key] = ws
    return ws


def groupnorm(x: torch.Tensor, samples: int, gamma: torch.Tensor, beta: torch.Tensor, eps: float, silu: bool,
              x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """GroupNorm(32) (+SiLU) over ``samples`` groups of rows; [x|x2] concatenated along channels.  When the GEMMs that produced x
    (and x2) left their partial sums (``_vc_gn``, see linear(gn_out=True)) the statistics pass is skipped: one read + one write.
    Reproducible mode: a sample is one frame, its statistics come from canonical leaves (groupnorm_canonical)."""
    if REPRODUCIBLE:
        return groupnorm_canonical(x, samples, x.shape[0] // samples, gamma, beta, eps, silu, x2=x2)
    _chk16(x, "groupnorm.x")
    rows, C1 = x.shape
    C2 = 0 if x2 is None else x2.shape[1]
    assert x.is_contiguous() and (x2 is None or x2.is_contiguous())
    out = torch.empty((rows, C1 + C2), device=x.device, dtype=torch.float16)
    p1, p2 = gn_part_of(x), (gn_part_of(x2) if x2 is not None else None)
    if p1 is not None and (x2 is None or p2 is not None) and (samples <= 4 or rows * (C1 + C2) * 2 >= GN_PARTS_MIN_MB * 1e6):
        cg = (C1 + C2) // 32
        g1 = p1.geom(samples, rows // samples)
        g2 = p2.geom(samples, rows // samples) if x2 is not None else None
        if g1 is not None and (x2 is None or g2 is not None) and cg % p1.sub == 0 and (x2 is None or (cg % p2.sub == 0 and C1 % p2.sub == 0)):
            lib = _lib.load()
            need = lib.vc_groupnorm_parts_ws_bytes(samples)
            key = (x.device, torch.cuda.current_stream().cuda_stream, "parts")
            ws = _gn_ws.get(key)
            if ws is None or ws.numel() < need:
                ws = torch.empty(max(need, 1 << 20), device=x.device, dtype=torch.uint8)
                _gn_ws[key] = ws
            global gn_from_parts_calls
            gn_from_parts_calls += 1
            check(lib.vc_groupnorm_from_parts(x.data_ptr(), C1, C.byref(g1), _ptr(x2), C2, C.byref(g2) if g2 is not None else None, samples,
                                              rows // samples, gamma.data_ptr(), beta.data_ptr(), eps, int(silu), out.data_ptr(), ws.data_ptr(),
                                              ws.numel(), _stream()), "vc_groupnorm_from_parts")
            return out
    ws = _gn_workspace(x.device, samples)
    check(_lib.load().vc_groupnorm_nhwc(x.data_ptr(), C1, _ptr(x2), C2, samples, rows // samples, gamma.data_ptr(), beta.data_ptr(),
                                        eps, int(silu), out.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "vc_groupnorm_nhwc")
    return out


def groupnorm_leaves(x: torch.Tensor, rows_per_leaf: int, x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 [rows / rows_per_leaf, 32, 2]: per-group (sum, sumsq) of every block of rows_per_leaf contiguous rows of [x|x2].  A leaf
    depends only on its rows, rows_per_leaf and the channel counts (one CTA per leaf, fixed order)."""
    _chk16(x, "groupnorm_leaves.x")
    rows, C1 = x.shape
    C2 = 0 if x2 is None else x2.shape[1]
    assert x.is_contiguous() and (x2 is None or x2.is_contiguous()) and rows % rows_per_leaf == 0
    leaves = torch.empty((rows // rows_per_leaf, 32, 2), device=x.device, dtype=torch.float32)
    check(_lib.load().vc_groupnorm_leaves(x.data_ptr(), C1, _ptr(x2), C2, rows // rows_per_leaf, rows_per_leaf, leaves.data_ptr(), _stream()),
          "vc_groupnorm_leaves")
    return leaves


def groupnorm_apply_leaves(x: torch.Tensor, samples: int, leaves: torch.Tensor, stat_rows: int, gamma: torch.Tensor, beta: torch.Tensor,
                           eps: float, silu: bool, x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Normalise ``samples`` groups of rows of [x|x2] with statistics = the sum, in index order, of each sample's share of the leaves
    ([samples * k, 32, 2], k consecutive leaves per sample) over ``stat_rows`` rows per sample."""
    _chk16(x, "groupnorm_apply_leaves.x")
    rows, C1 = x.shape
    C2 = 0 if x2 is None else x2.shape[1]
    assert leaves.dtype == torch.float32 and leaves.is_contiguous() and leaves.shape[0] % samples == 0
    out = torch.empty((rows, C1 + C2), device=x.device, dtype=torch.float16)
    ws = _gn_workspace(x.device, samples)
    check(_lib.load().vc_groupnorm_apply_leaves(x.data_ptr(), C1, _ptr(x2), C2, samples, rows // samples, leaves.data_ptr(),
                                                leaves.shape[0] // samples, stat_rows, gamma.data_ptr(), beta.data_ptr(), eps, int(silu),
                                                out.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "vc_groupnorm_apply_leaves")
    return out


def groupnorm_canonical(x: torch.Tensor, samples: int, hw: int, gamma: torch.Tensor, beta: torch.Tensor, eps: float, silu: bool,
                        x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """GroupNorm(32) (+SiLU) of ``samples`` groups of rows whose rows are (frame, pixel) with ``hw`` pixels per frame, from canonical
    leaves: every frame is cut into gn_leaf_chunks(hw) chunks, a leaf is (frame, chunk, group), and a sample's statistics are its leaves
    summed over frames, then chunks, in index order.  The result does not depend on how many samples the call holds, on the GPU
    count the frames are sharded over or on the SM count (hw = rows per sample: a per-frame GroupNorm)."""
    leaves = groupnorm_leaves(x, hw // gn_leaf_chunks(hw), x2=x2)
    return groupnorm_apply_leaves(x, samples, leaves, x.shape[0] // samples, gamma, beta, eps, silu, x2=x2)


def groupnorm_stats(x: torch.Tensor, samples: int) -> torch.Tensor:
    """Pass 1 of the split GroupNorm: fp32 [samples, 32, 2] = (sum, sumsq) per group over this rank's rows."""
    _chk16(x, "groupnorm_stats.x")
    rows, C1 = x.shape
    assert x.is_contiguous()
    stats = torch.empty((samples, 32, 2), device=x.device, dtype=torch.float32)
    ws = _gn_workspace(x.device, samples)
    check(_lib.load().vc_groupnorm_stats(x.data_ptr(), C1, None, 0, samples, rows // samples, stats.data_ptr(), ws.data_ptr(),
                                         ws.numel(), _stream()), "vc_groupnorm_stats")
    return stats


def groupnorm_apply(x: torch.Tensor, samples: int, stats: torch.Tensor, stat_rows: int, gamma: torch.Tensor, beta: torch.Tensor,
                    eps: float, silu: bool) -> torch.Tensor:
    """Pass 2: normalise with (all-reduced) statistics that cover ``stat_rows`` rows per sample."""
    _chk16(x, "groupnorm_apply.x")
    rows, C1 = x.shape
    out = torch.empty_like(x)
    check(_lib.load().vc_groupnorm_apply(x.data_ptr(), C1, None, 0, samples, rows // samples, stats.data_ptr(), stat_rows,
                                         gamma.data_ptr(), beta.data_ptr(), eps, int(silu), out.data_ptr(), _stream()), "vc_groupnorm_apply")
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    _chk16(x, "layernorm.x")
    assert x.is_contiguous()
    out = torch.empty_like(x)
    check(_lib.load().vc_layernorm(x.data_ptr(), x.shape[0], x.shape[1], gamma.data_ptr(), beta.data_ptr(), eps, out.data_ptr(),
                                   _stream()), "vc_layernorm")
    return out


def layernorm_stats(x: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """[M,2] fp32 (mean, rstd) per row: the statistics half of LayerNorm (the consumer GEMM applies them, see fold_layernorm)."""
    _chk16(x, "layernorm_stats.x")
    assert x.is_contiguous()
    stats = torch.empty((x.shape[0], 2), device=x.device, dtype=torch.float32)
    check(_lib.load().vc_layernorm_stats(x.data_ptr(), x.shape[0], x.shape[1], eps, stats.data_ptr(), _stream()), "vc_layernorm_stats")
    return stats


def softmax_rows(x: torch.Tensor, scale: float) -> torch.Tensor:
    """softmax(x*scale, dim=-1) of fp32 scores -> fp16."""
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2
    out = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    check(_lib.load().vc_softmax_rows_f32(x.data_ptr(), x.shape[0], x.shape[1], scale, out.data_ptr(), _stream()), "vc_softmax_rows_f32")
    return out


def _rows_view(x: torch.Tensor, rows: int, cols: int, who: str):
    """The kernels index a row matrix as base + row * stride(0) + column: reject views they would read or write past."""
    if x.dim() != 2 or x.shape[0] != rows or x.shape[1] < cols or x.stride(1) != 1 or x.stride(0) < x.shape[1]:
        raise VcError(f"{who}: expected a [{rows}, >= {cols}] row matrix with unit column stride, got shape {tuple(x.shape)} "
                      f"strides {x.stride()}")


def _dense16(x: torch.Tensor, rows: int, who: str):
    """fp16 [rows, C] rows packed densely (pitch C), 16-byte aligned, C a multiple of 8: the layout the uint4 kernels read."""
    _chk16(x, who)
    if x.dim() != 2 or x.shape[0] != rows or not x.is_contiguous() or x.shape[1] % 8 or x.data_ptr() % 16:
        raise VcError(f"{who}: expected a contiguous, 16-byte aligned fp16 [{rows}, C % 8 == 0] tensor, got shape {tuple(x.shape)} "
                      f"strides {x.stride()}")


def upsample2x(x: torch.Tensor, N: int, H: int, W: int) -> torch.Tensor:
    _dense16(x, N * H * W, "upsample.x")
    Cc = x.shape[1]
    out = torch.empty((N * 4 * H * W, Cc), device=x.device, dtype=torch.float16)
    check(_lib.load().vc_upsample2x_nhwc(x.data_ptr(), out.data_ptr(), N, H, W, Cc, _stream()), "vc_upsample2x_nhwc")
    return out


def im2col_s2(x: torch.Tensor, N: int, H: int, W: int, pad_lo: int = 1, pad_hi: Optional[int] = None) -> tuple:
    """stride-2 3x3 patches, zero padding pad_lo (top/left) and pad_hi (bottom/right; default = pad_lo).  U-Net Downsample:
    (1, 1); VAE Downsample: (0, 1) (ae_modules.py:102-106)."""
    _dense16(x, N * H * W, "im2col.x")
    Cc = x.shape[1]
    pad_hi = pad_lo if pad_hi is None else pad_hi
    Ho, Wo = (H + pad_lo + pad_hi - 3) // 2 + 1, (W + pad_lo + pad_hi - 3) // 2 + 1
    out = torch.empty((N * Ho * Wo, 9 * Cc), device=x.device, dtype=torch.float16)
    check(_lib.load().vc_im2col3x3_s2(x.data_ptr(), out.data_ptr(), N, H, W, Cc, pad_lo, Ho, Wo, _stream()), "vc_im2col3x3_s2")
    return out, Ho, Wo


def ncthw_to_rows(x: torch.Tensor, out: torch.Tensor, c_off: int = 0):
    """fp32 [B,C,T,H,W] -> fp16 rows [(B T H W), ld] at channel offset c_off ('b c t h w -> (b t) h w c').  Only the columns
    c_off .. c_off + C - 1 of out are written."""
    B, Cc, T, H, W = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    _chk16(out, "ncthw_to_rows.out")
    if c_off < 0:
        raise VcError(f"ncthw_to_rows: c_off {c_off} < 0")
    _rows_view(out, B * T * H * W, c_off + Cc, "ncthw_to_rows.out")
    check(_lib.load().vc_ncthw_f32_to_rows_f16(x.data_ptr(), out.data_ptr(), B, Cc, T, H * W, c_off, out.stride(0), _stream()),
          "vc_ncthw_f32_to_rows_f16")


def rows_to_ncthw(x: torch.Tensor, B: int, Cc: int, T: int, H: int, W: int) -> torch.Tensor:
    """The first Cc columns of fp32 rows [(B T H W), >= Cc] -> [B,C,T,H,W]."""
    if x.dtype != torch.float32 or not x.is_cuda:
        raise VcError(f"rows_to_ncthw.x: expected a CUDA fp32 tensor, got {x.dtype} on {x.device}")
    _rows_view(x, B * T * H * W, Cc, "rows_to_ncthw.x")
    out = torch.empty((B, Cc, T, H, W), device=x.device, dtype=torch.float32)
    check(_lib.load().vc_rows_f32_to_ncthw(x.data_ptr(), x.stride(0), out.data_ptr(), B, Cc, T, H * W, _stream()),
          "vc_rows_f32_to_ncthw")
    return out


def rows_f16_to_nchw(x: torch.Tensor, N: int, Cc: int, H: int, W: int) -> torch.Tensor:
    """The first Cc columns of fp16 rows [(N H W), >= Cc] -> fp32 [N,C,H,W]."""
    _chk16(x, "rows_f16_to_nchw.x")
    _rows_view(x, N * H * W, Cc, "rows_f16_to_nchw.x")
    out = torch.empty((N, Cc, H, W), device=x.device, dtype=torch.float32)
    check(_lib.load().vc_rows_f16_to_nchw_f32(x.data_ptr(), x.stride(0), out.data_ptr(), N, Cc, H * W, _stream()),
          "vc_rows_f16_to_nchw_f32")
    return out


def cast_f16(x: torch.Tensor) -> torch.Tensor:
    assert x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    check(_lib.load().vc_cast_f32_to_f16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "vc_cast_f32_to_f16")
    return out


def add_f16(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a + b of two contiguous fp16 tensors of one shape and an even element count (the kernel reads half2 pairs)."""
    _chk16(a, "add.a")
    _chk16(b, "add.b")
    if a.shape != b.shape or not (a.is_contiguous() and b.is_contiguous()) or a.numel() % 2 or (a.data_ptr() | b.data_ptr()) % 4:
        raise VcError(f"add_f16: expected two contiguous, 4-byte aligned fp16 tensors of one shape with an even element count, got "
                      f"{tuple(a.shape)} and {tuple(b.shape)}")
    out = torch.empty_like(a)
    check(_lib.load().vc_add_f16(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), _stream()), "vc_add_f16")
    return out


def gelu_f16(x: torch.Tensor) -> torch.Tensor:
    """exact-erf GELU, elementwise (nn.GELU() of the Resampler FeedForward, resampler.py:27-34)."""
    _chk16(x, "gelu.x")
    assert x.is_contiguous()
    out = torch.empty_like(x)
    check(_lib.load().vc_gelu_f16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "vc_gelu_f16")
    return out


# ----------------------------------------------------------------------------------------------------
# embedding MLP + DDIM update
# ----------------------------------------------------------------------------------------------------
def timestep_embedding(t: torch.Tensor, dim: int) -> torch.Tensor:
    assert t.dtype == torch.int64 and t.is_cuda
    out = torch.empty((t.shape[0], dim), device=t.device, dtype=torch.float32)
    check(_lib.load().vc_timestep_embedding(t.data_ptr(), t.shape[0], dim, out.data_ptr(), _stream()), "vc_timestep_embedding")
    return out


def small_linear(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], silu_in: bool = False,
                 add: Optional[torch.Tensor] = None) -> torch.Tensor:
    assert x.dtype == torch.float32 and w.dtype == torch.float32 and x.is_contiguous() and w.is_contiguous()
    out = torch.empty((x.shape[0], w.shape[0]), device=x.device, dtype=torch.float32)
    check(_lib.load().vc_small_linear_f32(x.data_ptr(), x.shape[0], x.shape[1], w.data_ptr(), _ptr(b), w.shape[0], int(silu_in),
                                          out.data_ptr(), _ptr(add), _stream()), "vc_small_linear_f32")
    return out


_ddim_ws = {}


def _update_args(x, v_uncond, sc: dict):
    """(vc_ddim_scalars, use_cfg, workspace) of one fused DDIM / DPM-Solver update: the step scalars `sc`, and the per-(device, stream)
    buffer of the per-block partial sums of the two std reductions."""
    s = DdimScalars()
    use_cfg = v_uncond is not None and sc["cfg_scale"] != 1.0
    s.cfg_scale, s.guidance_rescale = sc["cfg_scale"], sc["guidance_rescale"] if use_cfg else 0.0
    s.sqrt_ac_t, s.sqrt_1mac_t = sc["sqrt_ac_t"], sc["sqrt_1mac_t"]
    s.a_prev, s.sigma_t, s.scale_t, s.prev_scale_t = sc["a_prev"], sc["sigma_t"], sc["scale_t"], sc["prev_scale_t"]
    s.use_cfg = int(use_cfg)
    s.reproducible = int(REPRODUCIBLE)
    key = (x.device, torch.cuda.current_stream().cuda_stream)
    ws = _ddim_ws.get(key)
    if ws is None:
        ws = torch.zeros(4 * 1025, device=x.device, dtype=torch.float64)
        _ddim_ws[key] = ws
    return s, use_cfg, ws


def ddim_update(x, v_cond, v_uncond, noise, sc: dict, v_uncond_img=None, cfg_img: float = 0.0):
    """Fused ddim.py:228-281.  sc: cfg_scale, guidance_rescale, sqrt_ac_t, sqrt_1mac_t, a_prev, sigma_t, scale_t, prev_scale_t.
    v_uncond_img / cfg_img: the third ("image, no text") branch of ddim_multiplecond.py:227-233."""
    for t in (x, v_cond, noise) + ((v_uncond_img,) if v_uncond_img is not None else ()):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda
    s, use_cfg, ws = _update_args(x, v_uncond, sc)
    x_prev, pred_x0 = torch.empty_like(x), torch.empty_like(x)
    if v_uncond_img is not None and use_cfg:
        check(_lib.load().vc_ddim_update3(x.data_ptr(), v_cond.data_ptr(), v_uncond.data_ptr(), v_uncond_img.data_ptr(), float(cfg_img),
                                          noise.data_ptr(), x_prev.data_ptr(), pred_x0.data_ptr(), x.numel(), C.byref(s), ws.data_ptr(),
                                          _stream()), "vc_ddim_update3")
        return x_prev, pred_x0
    check(_lib.load().vc_ddim_update(x.data_ptr(), v_cond.data_ptr(), _ptr(v_uncond) if use_cfg else None, noise.data_ptr(),
                                     x_prev.data_ptr(), pred_x0.data_ptr(), x.numel(), C.byref(s), ws.data_ptr(), _stream()),
          "vc_ddim_update")
    return x_prev, pred_x0


_FRAME_KEYS = ("sqrt_ac_t", "sqrt_1mac_t", "a_prev", "sigma_t", "scale_t", "prev_scale_t")


def ddim_update_frames(x, v_cond, v_uncond, noise, sc: dict, frames, v_uncond_img=None, cfg_img: float = 0.0):
    """ddim_update with a step per frame (vc_ddim_update_frames): x and the predictions are [B', C, T, H, W] fp32 and frame t takes the
    step scalars frames[t] (a dict with sqrt_ac_t, sqrt_1mac_t, a_prev, sigma_t, scale_t, prev_scale_t); sc holds the per-call
    cfg_scale and guidance_rescale.  The guidance-rescale stds run over the whole input, as in ddim_update.  T <= 128.  With every
    frames[t] equal to sc's step scalars the result is ddim_update's bit for bit.  Returns (x_prev, pred_x0)."""
    for t in (x, v_cond, noise) + ((v_uncond_img,) if v_uncond_img is not None else ()):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda and t.shape == x.shape
    if x.dim() != 5 or len(frames) != x.shape[2]:
        raise VcError(f"ddim_update_frames: x must be [B, C, T, H, W] with one entry of `frames` per frame, got {tuple(x.shape)} and "
                      f"{len(frames)} entries")
    T, HW = x.shape[2], x.shape[3] * x.shape[4]
    if T > _lib.DDIM_MAX_FRAMES:
        raise VcError(f"ddim_update_frames: T={T} unsupported (1..{_lib.DDIM_MAX_FRAMES})")
    s, use_cfg, ws = _update_args(x, v_uncond, dict(sc, **{k: 0.0 for k in _FRAME_KEYS}))
    tab = (_lib.DdimFrameScalars * T)(*(_lib.DdimFrameScalars(*(f[k] for k in _FRAME_KEYS)) for f in frames))
    x_prev, pred_x0 = torch.empty_like(x), torch.empty_like(x)
    vi = v_uncond_img if use_cfg else None
    check(_lib.load().vc_ddim_update_frames(x.data_ptr(), v_cond.data_ptr(), _ptr(v_uncond) if use_cfg else None, _ptr(vi),
                                            float(cfg_img), noise.data_ptr(), x_prev.data_ptr(), pred_x0.data_ptr(), x.numel(), T, HW,
                                            C.byref(s), tab, ws.data_ptr(), _stream()), "vc_ddim_update_frames")
    return x_prev, pred_x0


def dpm_update(x, v_cond, v_uncond, noise, sc: dict, x0_hist, v_uncond_img=None, cfg_img: float = 0.0):
    """One DPM-Solver++(2M) step (vc_dpm_update): ddim_update's x_{t-1}, plus sc["c_hist"] * (x0 - x0_hist) where x0 is this step's x0
    prediction before the dynamic rescale.  x0_hist (fp32, x's shape) holds the previous step's x0, is read only when c_hist != 0 and
    is overwritten in place with this step's.  Returns (x_prev, pred_x0) like ddim_update."""
    for t in (x, v_cond, noise, x0_hist) + ((v_uncond_img,) if v_uncond_img is not None else ()):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda
    assert x0_hist.shape == x.shape
    s, use_cfg, ws = _update_args(x, v_uncond, sc)
    x_prev, pred_x0 = torch.empty_like(x), torch.empty_like(x)
    vi = v_uncond_img if use_cfg else None
    check(_lib.load().vc_dpm_update(x.data_ptr(), v_cond.data_ptr(), _ptr(v_uncond) if use_cfg else None, _ptr(vi), float(cfg_img),
                                    noise.data_ptr(), x0_hist.data_ptr(), x_prev.data_ptr(), pred_x0.data_ptr(), x.numel(), C.byref(s),
                                    float(sc["c_hist"]), ws.data_ptr(), _stream()), "vc_dpm_update")
    return x_prev, pred_x0


def dpm3_update(x, v_cond, v_uncond, noise, sc: dict, x0_hist1, x0_hist2, v_uncond_img=None, cfg_img: float = 0.0):
    """One DPM-Solver++(3M) SDE step (vc_dpm3_update): ddim_update's x_{t-1} (eta = 1), plus sc["c1"] * (x0 - x0_hist1) +
    sc["c2"] * (x0_hist1 - x0_hist2), where x0 is this step's x0 prediction before the dynamic rescale.  x0_hist1 / x0_hist2 (fp32,
    x's shape) hold the previous step's x0 and the one before; a term whose coefficient is 0 reads nothing.  x0_hist1 is only read and
    x0_hist2 is overwritten in place with this step's x0, so the caller swaps the two after each step.  sc["c2"] = 0 gives dpm_update's
    x_prev with c_hist = sc["c1"] bit for bit.  Returns (x_prev, pred_x0) like ddim_update."""
    for t in (x, v_cond, noise, x0_hist1, x0_hist2) + ((v_uncond_img,) if v_uncond_img is not None else ()):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda
    assert x0_hist1.shape == x.shape and x0_hist2.shape == x.shape
    s, use_cfg, ws = _update_args(x, v_uncond, sc)
    x_prev, pred_x0 = torch.empty_like(x), torch.empty_like(x)
    vi = v_uncond_img if use_cfg else None
    check(_lib.load().vc_dpm3_update(x.data_ptr(), v_cond.data_ptr(), _ptr(v_uncond) if use_cfg else None, _ptr(vi), float(cfg_img),
                                     noise.data_ptr(), x0_hist1.data_ptr(), x0_hist2.data_ptr(), x_prev.data_ptr(), pred_x0.data_ptr(),
                                     x.numel(), C.byref(s), float(sc["c1"]), float(sc["c2"]), ws.data_ptr(), _stream()), "vc_dpm3_update")
    return x_prev, pred_x0
