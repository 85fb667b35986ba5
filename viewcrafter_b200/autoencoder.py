"""Drop-in ``AutoencoderKL`` (reference: lvdm/models/autoencoder.py:13-107, lvdm/modules/networks/ae_modules.py).

``decode(z)`` -- the hot-path half -- runs on the sm_90a kernels: post_quant 1x1 GEMM, conv_in, ResnetBlocks
(GroupNorm+swish kernel, 9-tap wgmma GEMMs, 1x1 nin_shortcut fused as residual), the single-head d=512 AttnBlock
(QK^T and PV as wgmma GEMMs around a row-softmax kernel), nearest-2x upsample + conv, GroupNorm+swish, conv_out.
State-dict keys match the reference (``post_quant_conv.*``, ``decoder.*``, ``encoder.*``, ``quant_conv.*``).
``encode(x)`` (conditioning renders, once per clip; SURVEY.md 8f rank f1) runs the Encoder on the same kernels: the stride-2
Downsample (zero-pad right/bottom, ae_modules.py:102-106) is an im2col + GEMM, and conv_out is folded with the 1x1 quant_conv;
it returns the reference's ``DiagonalGaussianDistribution`` over fp32 moments.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .distributions import DiagonalGaussianDistribution, posterior_class


def _gn(c):
    return nn.GroupNorm(32, c, eps=1e-6, affine=True)


class _VResnet(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.norm1, self.conv1 = _gn(cin), nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2, self.conv2 = _gn(cout), nn.Conv2d(cout, cout, 3, padding=1)
        if cin != cout:
            self.nin_shortcut = nn.Conv2d(cin, cout, 1)


class _VAttn(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.norm = _gn(c)
        self.q, self.k, self.v, self.proj_out = (nn.Conv2d(c, c, 1) for _ in range(4))


class _VUpsample(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)


class _VDownsample(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=0)


class Decoder(nn.Module):
    """Parameter tree of ae_modules.Decoder (:466-537)."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0, resamp_with_conv=True,
                 in_channels, resolution, z_channels, give_pre_end=False, tanh_out=False, use_linear_attn=False,
                 attn_type="vanilla", **ignored):
        super().__init__()
        if use_linear_attn or attn_type != "vanilla" or give_pre_end or tanh_out or not resamp_with_conv:
            raise NotImplementedError("viewcrafter_b200 Decoder: option not used by the ViewCrafter VAE")
        n = len(ch_mult)
        cur = ch * ch_mult[-1]
        res = resolution // 2 ** (n - 1)
        self.conv_in = nn.Conv2d(z_channels, cur, 3, padding=1)
        self.mid = nn.Module()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = _VResnet(cur, cur), _VAttn(cur), _VResnet(cur, cur)
        self.up = nn.ModuleList()
        for lvl in reversed(range(n)):
            stage = nn.Module()
            stage.block, stage.attn = nn.ModuleList(), nn.ModuleList()
            cout = ch * ch_mult[lvl]
            for _ in range(num_res_blocks + 1):
                stage.block.append(_VResnet(cur, cout))
                cur = cout
                if res in attn_resolutions:
                    stage.attn.append(_VAttn(cur))
            if lvl != 0:
                stage.upsample = _VUpsample(cur)
                res *= 2
            self.up.insert(0, stage)
        self.norm_out = _gn(cur)
        self.conv_out = nn.Conv2d(cur, out_ch, 3, padding=1)


class Encoder(nn.Module):
    """Parameter tree of ae_modules.Encoder (:364-463) so the full checkpoint loads; compute is next-tier."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0, resamp_with_conv=True,
                 in_channels, resolution, z_channels, double_z=True, use_linear_attn=False, attn_type="vanilla", **ignored):
        super().__init__()
        n = len(ch_mult)
        self.conv_in = nn.Conv2d(in_channels, ch, 3, padding=1)
        res = resolution
        in_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        cur = ch
        for lvl in range(n):
            stage = nn.Module()
            stage.block, stage.attn = nn.ModuleList(), nn.ModuleList()
            cur, cout = ch * in_mult[lvl], ch * ch_mult[lvl]
            for _ in range(num_res_blocks):
                stage.block.append(_VResnet(cur, cout))
                cur = cout
                if res in attn_resolutions:
                    stage.attn.append(_VAttn(cur))
            if lvl != n - 1:
                stage.downsample = _VDownsample(cur)
                res //= 2
            self.down.append(stage)
        self.mid = nn.Module()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = _VResnet(cur, cur), _VAttn(cur), _VResnet(cur, cur)
        self.norm_out = _gn(cur)
        self.conv_out = nn.Conv2d(cur, 2 * z_channels if double_z else z_channels, 3, padding=1)


class AutoencoderKL(nn.Module):
    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, ckpt_path=None, ignore_keys=[], image_key="image",
                 colorize_nlabels=None, monitor=None, test=False, logdir=None, input_dim=4, test_args=None):
        super().__init__()
        assert ddconfig["double_z"]
        self.image_key = image_key
        self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        self.loss = nn.Identity()
        self.quant_conv = nn.Conv2d(2 * ddconfig["z_channels"], 2 * embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, ddconfig["z_channels"], 1)
        self.embed_dim, self.input_dim = embed_dim, input_dim
        self._packed = None
        self._packed_enc = None
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packed())
        if ckpt_path is not None:
            sd = torch.load(ckpt_path, map_location="cpu")
            self.load_state_dict(sd.get("state_dict", sd), strict=False)

    def invalidate_packed(self):
        self._packed = None
        self._packed_enc = None

    def _apply(self, fn, *a, **k):
        # a pure device move carries the packed kernel operands along; a dtype change drops them (cf. UNetModel._apply)
        keep = ops.is_device_only(fn)
        packed, packed_enc = (self._packed, self._packed_enc) if keep else (None, None)
        self._packed = None
        self._packed_enc = None
        r = super()._apply(fn, *a, **k)
        if packed is not None:
            self._packed = ops.tree_apply(packed, fn)
        if packed_enc is not None:
            self._packed_enc = ops.tree_apply(packed_enc, fn)
        return r

    @property
    def device(self):
        return self.post_quant_conv.weight.device

    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _f32(t):
        return t.detach().float().contiguous()

    def _pack_res(self, m: _VResnet):
        f = self._f32
        P = dict(gn1=(f(m.norm1.weight), f(m.norm1.bias)), w1=ops.pack_conv3x3(m.conv1.weight.detach()), b1=f(m.conv1.bias),
                 gn2=(f(m.norm2.weight), f(m.norm2.bias)), w2=ops.pack_conv3x3(m.conv2.weight.detach()), b2=f(m.conv2.bias))
        if hasattr(m, "nin_shortcut"):
            P["skip_w"], P["skip_b"] = ops.pack_linear(m.nin_shortcut.weight.detach()), f(m.nin_shortcut.bias)
        return P

    def _pack_attn(self, m: _VAttn):
        f = self._f32
        return dict(gn=(f(m.norm.weight), f(m.norm.bias)),
                    qk_w=torch.cat([ops.pack_linear(m.q.weight.detach()), ops.pack_linear(m.k.weight.detach())], 0).contiguous(),
                    qk_b=torch.cat([f(m.q.bias), f(m.k.bias)]).contiguous(),
                    v_w=ops.pack_linear(m.v.weight.detach()), v_b=f(m.v.bias),
                    o_w=ops.pack_linear(m.proj_out.weight.detach()), o_b=f(m.proj_out.bias))

    def _pack(self):
        f = self._f32
        d = self.decoder
        zc = self.post_quant_conv.weight.shape[1]
        pq = torch.zeros(self.post_quant_conv.weight.shape[0], 8, device=self.device)
        pq[:, :zc] = self.post_quant_conv.weight.detach().reshape(-1, zc)
        P = dict(pq_w=pq.to(torch.float16).contiguous(), pq_b=f(self.post_quant_conv.bias),
                 in_w=ops.pack_conv3x3(d.conv_in.weight.detach(), k_pad=8), in_b=f(d.conv_in.bias),
                 mid1=self._pack_res(d.mid.block_1), attn=self._pack_attn(d.mid.attn_1), mid2=self._pack_res(d.mid.block_2))
        ups = []
        for stage in d.up:
            S = dict(blocks=[self._pack_res(b) for b in stage.block], attns=[self._pack_attn(a) for a in stage.attn])
            if hasattr(stage, "upsample"):
                S["up_w"], S["up_b"] = ops.pack_upconv3x3(stage.upsample.conv.weight.detach()), f(stage.upsample.conv.bias)
            ups.append(S)
        P["up"] = ups
        P["out_gn"] = (f(d.norm_out.weight), f(d.norm_out.bias))
        P["out_w"], P["out_b"] = ops.pack_conv3x3(d.conv_out.weight.detach()), f(d.conv_out.bias)
        self._packed = P
        return P

    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _res(P, x, N, H, W):
        a = ops.groupnorm(x, N, *P["gn1"], 1e-6, True)
        h = ops.conv3x3(a, N, H, W, P["w1"], bias=P["b1"])
        b = ops.groupnorm(h, N, *P["gn2"], 1e-6, True)
        xs = ops.linear(x, P["skip_w"], bias=P["skip_b"]) if "skip_w" in P else x
        return ops.conv3x3(b, N, H, W, P["w2"], bias=P["b2"], res=xs)

    @staticmethod
    def _attn(P, x, N, H, W):
        """AttnBlock (ae_modules.py:53-78): softmax(q k^T C^-0.5) v, single head of width C, per image."""
        HW, C = H * W, x.shape[1]
        hn = ops.groupnorm(x, N, *P["gn"], 1e-6, False)
        qk = ops.linear(hn, P["qk_w"], bias=P["qk_b"])                                   # [N*HW, 2C]
        out = torch.empty_like(x)
        HWp = (HW + 7) // 8 * 8            # the key axis is a GEMM reduction / row pitch: TMA needs 16-byte multiples
        for n in range(N):
            rows = slice(n * HW, (n + 1) * HW)
            kn, hv = qk[rows, C:], hn[rows]
            if HWp != HW:                                                                 # odd token counts (e.g. a 5x9 latent): zero key rows,
                kn = torch.zeros((HWp, C), device=x.device, dtype=torch.float16); kn[:HW] = qk[rows, C:]
                hv = torch.zeros((HWp, C), device=x.device, dtype=torch.float16); hv[:HW] = hn[rows]
            s = ops.linear(qk[rows, :C], kn, out_f32=True)                                # S = Q K^T  [HW, HWp] fp32
            if HWp != HW:
                s[:, HW:] = float("-inf")                                                 # ... masked out of the softmax
            p = ops.softmax_rows(s, float(C) ** -0.5)                                     # fp16 probabilities
            vt = ops.linear(P["v_w"], hv)                                                 # V^T (bias folded below) [C, HWp]
            o = ops.linear(p, vt, bias=P["v_b"])                                          # P V + b_v  (rows of P sum to 1)
            ops.linear(o, P["o_w"], bias=P["o_b"], res=x[rows], out=out[rows])
        return out

    @torch.no_grad()
    def decode(self, z, **kwargs):
        """z [N, z_channels, h, w] -> [N, out_ch, 8h, 8w] in z.dtype (autoencoder.py:104-107, ae_modules.py:539-578)."""
        ops.require_cuda(z.device, "viewcrafter_b200.AutoencoderKL.decode")
        P = self._packed or self._pack()
        N, zc, H, W = z.shape
        rows = torch.zeros((N * H * W, 8), device=z.device, dtype=torch.float16)
        ops.ncthw_to_rows(z.float().contiguous().reshape(N, zc, 1, H, W), rows, 0)
        zq = torch.zeros((N * H * W, 8), device=z.device, dtype=torch.float16)
        ops.linear(rows, P["pq_w"], bias=P["pq_b"], out=zq)                               # post_quant_conv, writes 4 of 8 columns
        h = ops.conv3x3(zq, N, H, W, P["in_w"], bias=P["in_b"])
        h = self._res(P["mid1"], h, N, H, W)
        h = self._attn(P["attn"], h, N, H, W)
        h = self._res(P["mid2"], h, N, H, W)
        for S in reversed(P["up"]):
            for i, B in enumerate(S["blocks"]):
                h = self._res(B, h, N, H, W)
                if S["attns"]:
                    h = self._attn(S["attns"][i], h, N, H, W)
            if "up_w" in S:
                h = ops.upconv3x3(h, N, H, W, S["up_w"], bias=S["up_b"])                # upsample folded into four parity sub-convolutions
                H, W = 2 * H, 2 * W
        y = ops.conv3x3(ops.groupnorm(h, N, *P["out_gn"], 1e-6, True), N, H, W, P["out_w"], bias=P["out_b"], out_f32=True)
        oc = y.shape[1]
        return ops.rows_to_ncthw(y, N, oc, 1, H, W).reshape(N, oc, H, W).to(z.dtype)

    # ------------------------------------------------------------------------------------------
    def _pack_encoder(self):
        f = self._f32
        e = self.encoder
        P = dict(in_w=ops.pack_conv3x3(e.conv_in.weight.detach(), k_pad=8), in_b=f(e.conv_in.bias),
                 mid1=self._pack_res(e.mid.block_1), attn=self._pack_attn(e.mid.attn_1), mid2=self._pack_res(e.mid.block_2))
        downs = []
        for stage in e.down:
            S = dict(blocks=[self._pack_res(b) for b in stage.block], attns=[self._pack_attn(a) for a in stage.attn])
            if hasattr(stage, "downsample"):
                w = stage.downsample.conv.weight.detach()                                  # [C, C, 3, 3] -> [C, 9*C] tap-major
                S["down_w"] = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(torch.float16).contiguous()
                S["down_b"] = f(stage.downsample.conv.bias)
            downs.append(S)
        P["down"] = downs
        P["out_gn"] = (f(e.norm_out.weight), f(e.norm_out.bias))
        # conv_out (3x3, C -> 2z) followed by the 1x1 quant_conv (2z -> 2*embed) is one 3x3 conv with the combined weights
        # W[o] = sum_m Wq[o, m] * Wc[m],  b = Wq bc + bq   (autoencoder.py:99-100): one GEMM, one rounding of the weights
        wq = self.quant_conv.weight.detach().float().reshape(self.quant_conv.weight.shape[0], -1)      # [2e, 2z]
        wc = e.conv_out.weight.detach().float()                                                         # [2z, C, 3, 3]
        w = torch.einsum("om,mchw->ochw", wq, wc)
        P["out_w"] = ops.pack_conv3x3(w)
        P["out_b"] = (wq @ e.conv_out.bias.detach().float() + self.quant_conv.bias.detach().float()).contiguous()
        self._packed_enc = P
        return P

    @torch.no_grad()
    def encode_moments(self, x):
        """x [N, in_channels, H, W] (H, W multiples of 2^(levels-1)) -> fp32 moments [N, 2*embed_dim, H/8, W/8]
        (autoencoder.py:97-100, ae_modules.py:430-463)."""
        ops.require_cuda(x.device, "viewcrafter_b200.AutoencoderKL.encode")
        P = self._packed_enc or self._pack_encoder()
        N, Cin, H, W = x.shape
        nd = len(P["down"]) - 1
        if H % (1 << nd) or W % (1 << nd):
            raise ValueError(f"AutoencoderKL.encode: H, W must be multiples of {1 << nd}, got {H}x{W}")
        rows = torch.zeros((N * H * W, 8), device=x.device, dtype=torch.float16)
        ops.ncthw_to_rows(x.float().contiguous().reshape(N, Cin, 1, H, W), rows, 0)
        h = ops.conv3x3(rows, N, H, W, P["in_w"], bias=P["in_b"])
        for S in P["down"]:
            for i, B in enumerate(S["blocks"]):
                h = self._res(B, h, N, H, W)
                if S["attns"]:
                    h = self._attn(S["attns"][i], h, N, H, W)
            if "down_w" in S:
                cols, H, W = ops.im2col_s2(h, N, H, W, pad_lo=0, pad_hi=1)
                h = ops.linear(cols, S["down_w"], bias=S["down_b"])
        h = self._res(P["mid1"], h, N, H, W)
        h = self._attn(P["attn"], h, N, H, W)
        h = self._res(P["mid2"], h, N, H, W)
        y = ops.conv3x3(ops.groupnorm(h, N, *P["out_gn"], 1e-6, True), N, H, W, P["out_w"], bias=P["out_b"], out_f32=True)
        oc = y.shape[1]
        return ops.rows_to_ncthw(y, N, oc, 1, H, W).reshape(N, oc, H, W)

    def encode(self, x, **kwargs):
        """-> DiagonalGaussianDistribution(moments)  (autoencoder.py:97-102); moments are fp32."""
        return posterior_class()(self.encode_moments(x))
