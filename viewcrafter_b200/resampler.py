"""Drop-in ``Resampler`` / ``ImageProjModel`` (reference: lvdm/modules/encoders/resampler.py:9-145) -- SURVEY.md 8(f) rank f3.

``image_proj_model`` of the ViewCrafter checkpoints (configs/inference_pvd_1024.yaml:100-111): the CLIP image tokens
``[B, 257, 1280]`` are turned into the ``num_queries * video_length`` image-context tokens ``[B, 256, 1024]`` that the
U-Net's image cross-attention consumes (utils/diffusion_utils.py:128-129,149-150; twice per clip).  Same constructor
kwargs, ``forward`` signature and state-dict keys (``latents``, ``proj_in``, ``proj_out``, ``norm_out``,
``layers.{i}.0.{norm1,norm2,to_q,to_kv,to_out}``, ``layers.{i}.1.{0,1,3}``) as the reference; the forward runs on the
same CUDA kernels as the U-Net: wgmma tap-GEMM for every Linear (residual adds fused into the epilogue), the d=64
flash-attention kernel for PerceiverAttention (scale = dim_head**-0.25 applied to q and k = dim_head**-0.5 on the
scores), LayerNorm rows, exact-erf GELU.  No CPU path (ops.require_cuda).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops


class ImageProjModel(nn.Module):
    """Linear(clip_embeddings_dim -> tokens * dim) + LayerNorm (resampler.py:9-24); not used by the shipped configs."""

    def __init__(self, cross_attention_dim=1024, clip_embeddings_dim=1024, clip_extra_context_tokens=4):
        super().__init__()
        self.cross_attention_dim = cross_attention_dim
        self.clip_extra_context_tokens = clip_extra_context_tokens
        self.proj = nn.Linear(clip_embeddings_dim, clip_extra_context_tokens * cross_attention_dim)
        self.norm = nn.LayerNorm(cross_attention_dim)

    @torch.no_grad()
    def forward(self, image_embeds):
        ops.require_cuda(self.proj.weight.device, "viewcrafter_b200.ImageProjModel")
        x = ops.cast_f16(image_embeds.reshape(-1, image_embeds.shape[-1]).float().contiguous())
        y = ops.linear(x, ops.pack_linear(self.proj.weight.detach()), bias=self.proj.bias.detach().float().contiguous())
        y = ops.layernorm(y.reshape(-1, self.cross_attention_dim), self.norm.weight.detach().float().contiguous(),
                          self.norm.bias.detach().float().contiguous())
        return y.reshape(-1, self.clip_extra_context_tokens, self.cross_attention_dim).to(image_embeds.dtype)


def _feed_forward(dim, mult=4):
    inner = int(dim * mult)
    return nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, inner, bias=False), nn.GELU(), nn.Linear(inner, dim, bias=False))


class _PerceiverAttention(nn.Module):
    """Parameter holder with the reference's names (resampler.py:48-60)."""

    def __init__(self, *, dim, dim_head=64, heads=8):
        super().__init__()
        self.dim_head, self.heads = dim_head, heads
        inner = dim_head * heads
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_kv = nn.Linear(dim, inner * 2, bias=False)
        self.to_out = nn.Linear(inner, dim, bias=False)


class Resampler(nn.Module):
    def __init__(self, dim=1024, depth=8, dim_head=64, heads=16, num_queries=8, embedding_dim=768, output_dim=1024,
                 ff_mult=4, video_length=None):
        super().__init__()
        if dim_head != 64:
            raise NotImplementedError("viewcrafter_b200.Resampler: the attention kernel is built for dim_head == 64")
        if dim % 8 or embedding_dim % 8 or output_dim % 8:
            raise NotImplementedError("viewcrafter_b200.Resampler: widths must be multiples of 8 (16-byte TMA strides)")
        self.num_queries = num_queries
        self.video_length = video_length
        if video_length is not None:
            num_queries = num_queries * video_length
        self.latents = nn.Parameter(torch.randn(1, num_queries, dim) / dim ** 0.5)
        self.proj_in = nn.Linear(embedding_dim, dim)
        self.proj_out = nn.Linear(dim, output_dim)
        self.norm_out = nn.LayerNorm(output_dim)
        self.layers = nn.ModuleList([nn.ModuleList([_PerceiverAttention(dim=dim, dim_head=dim_head, heads=heads),
                                                    _feed_forward(dim=dim, mult=ff_mult)]) for _ in range(depth)])
        self.heads = heads
        self._packed = None
        # fires for a load through any ancestor too (VIPLatentDiffusion.load_state_dict, diffusion_utils.py:83-108)
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packed())

    # weights are packed (fp16, K-contiguous) once per load / device move
    def invalidate_packed(self):
        self._packed = None

    def _apply(self, fn, *a, **k):
        self._packed = None
        return super()._apply(fn, *a, **k)

    def _pack(self):
        ops.require_cuda(self.latents.device, "viewcrafter_b200.Resampler")
        f = lambda t: t.detach().float().contiguous()
        P = dict(latents=ops.cast_f16(f(self.latents[0])),
                 in_w=ops.pack_linear(self.proj_in.weight.detach()), in_b=f(self.proj_in.bias),
                 out_w=ops.pack_linear(self.proj_out.weight.detach()), out_b=f(self.proj_out.bias),
                 out_ln=(f(self.norm_out.weight), f(self.norm_out.bias)), layers=[])
        for attn, ff in self.layers:
            P["layers"].append(dict(
                ln1=(f(attn.norm1.weight), f(attn.norm1.bias)), ln2=(f(attn.norm2.weight), f(attn.norm2.bias)),
                q_w=ops.pack_linear(attn.to_q.weight.detach()), kv_w=ops.pack_linear(attn.to_kv.weight.detach()),
                o_w=ops.pack_linear(attn.to_out.weight.detach()),
                ff_ln=(f(ff[0].weight), f(ff[0].bias)), ff1_w=ops.pack_linear(ff[1].weight.detach()),
                ff2_w=ops.pack_linear(ff[3].weight.detach())))
        self._packed = P
        return P

    @torch.no_grad()
    def forward(self, x):
        """x [B, n1, embedding_dim] -> [B, num_queries(*video_length), output_dim] in x.dtype (resampler.py:134-145)."""
        P = self._packed or self._pack()
        B, n1, E = x.shape
        L, D = P["latents"].shape
        inner = self.heads * 64
        xr = ops.linear(ops.cast_f16(x.reshape(B * n1, E).float().contiguous()), P["in_w"], bias=P["in_b"])     # proj_in
        lat = P["latents"].repeat(B, 1)                                                                        # [B*L, D]
        nk = n1 + L
        for Q in P["layers"]:
            # PerceiverAttention (resampler.py:62-94): keys/values over cat(norm1(x), norm2(latents)), queries = norm2(latents)
            xn = ops.layernorm(xr, *Q["ln1"])
            ln = ops.layernorm(lat, *Q["ln2"])
            kv_in = torch.empty((B * nk, D), device=lat.device, dtype=torch.float16)
            kv3 = kv_in.view(B, nk, D)
            kv3[:, :n1] = xn.view(B, n1, D)
            kv3[:, n1:] = ln.view(B, L, D)
            q = ops.linear(ln, Q["q_w"])
            kv = ops.linear(kv_in, Q["kv_w"])                                                                   # [B*nk, 2*inner]
            a = ops.flash_attn(q, kv[:, :inner], kv[:, inner:], B, L, nk, self.heads, scale=0.125)
            lat = ops.linear(a, Q["o_w"], res=lat)                                                              # + latents
            # FeedForward (resampler.py:27-34): LN, Linear, GELU(erf), Linear, + latents
            h = ops.linear(ops.layernorm(lat, *Q["ff_ln"]), Q["ff1_w"])
            lat = ops.linear(ops.gelu_f16(h), Q["ff2_w"], res=lat)
        y = ops.layernorm(ops.linear(lat, P["out_w"], bias=P["out_b"]), *P["out_ln"])
        return y.view(B, L, -1).to(x.dtype)
