"""Executes the parameter containers of `layers.py` on the sm_90a kernels.

Activation layout: 2-D tensors [rows, C] with rows ordered (batch b, frame t, y, x) — i.e. channels-last
[B, T, H, W, C].  The reference's `(b t) c h w  <->  b c t h w  <->  (b h w) t c` permutes
(diffusers TemporalConvLayer / TransformerTemporalModel forward) are never materialised: frame-wise ops view the rows
as B*T images, temporal ops as B volumes, token-wise ops as a flat matrix.

Weights are converted once per (dtype, device) into the layouts the kernels want:
  conv 3x3   [Cout, Cin, 3, 3]    -> [Cout, 9*Cin]  (tap-major: r, s, c)
  conv (3,1,1) [Cout, Cin, 3,1,1] -> [Cout, 3*Cin]
  to_q/to_k/to_v                  -> one fused [3*inner, C] matrix (self-attention) / [2*inner, Ckv] (cross K,V)
  biases, norm gains              -> fp32
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn as nn

from . import layers as L
from . import ops


@dataclass
class Geo:
    b: int      # batch (CFG halves x prompts)
    t: int      # frames incl. the condition frame
    h: int
    w: int

    @property
    def n(self):
        return self.b * self.t

    @property
    def hw(self):
        return self.h * self.w

    @property
    def rows(self):
        return self.b * self.t * self.h * self.w

    def down(self):
        # conv 3x3, stride 2, padding 1: ceil(h / 2)
        return Geo(self.b, self.t, (self.h + 1) // 2, (self.w + 1) // 2)

    def up(self):
        return Geo(self.b, self.t, self.h * 2, self.w * 2)


# ------------------------------------------------------------------------------------------------ weight prep
def _f32(t: Optional[torch.Tensor]):
    return None if t is None else t.detach().float().contiguous()


def _w(t: torch.Tensor, dtype):
    return t.detach().to(dtype).contiguous()


def prep_linear(lin: nn.Linear, dtype):
    return _w(lin.weight, dtype), _f32(lin.bias)


def prep_conv3x3(conv: nn.Conv2d, dtype, pad_cin_to: Optional[int] = None):
    w = conv.weight.detach()
    if pad_cin_to is not None and w.shape[1] < pad_cin_to:
        wp = torch.zeros((w.shape[0], pad_cin_to, 3, 3), device=w.device, dtype=w.dtype)
        wp[:, : w.shape[1]] = w
        w = wp
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(dtype).contiguous(), _f32(conv.bias)


def prep_conv1x1(conv: nn.Conv2d, dtype):
    return _w(conv.weight.reshape(conv.weight.shape[0], -1), dtype), _f32(conv.bias)


def prep_conv3d_t(conv: nn.Conv3d, dtype):
    w = conv.weight.detach()
    co, ci = w.shape[0], w.shape[1]
    return w.reshape(co, ci, 3).permute(0, 2, 1).reshape(co, 3 * ci).to(dtype).contiguous(), _f32(conv.bias)


def prep_norm(norm):
    return _f32(norm.weight), _f32(norm.bias)


_prepared_generation = 0


class Prepared:
    """Per-model cache: module -> dict of kernel-layout tensors.  `gen` is a process-wide generation number: anything
    that holds raw pointers into these tensors (captured CUDA graphs) keys itself on it, because `id()` of a freed
    object can be re-used."""

    def __init__(self, dtype, device):
        global _prepared_generation
        _prepared_generation += 1
        self.gen = _prepared_generation
        self.dtype = dtype
        self.device = device
        self.m: Dict[int, dict] = {}

    def get(self, mod) -> dict:
        return self.m[id(mod)]

    def put(self, mod, d: dict):
        self.m[id(mod)] = d
        return d


def prepare_module(prep: Prepared, mod: nn.Module):
    """Recursively convert the weights of every known container under `mod`."""
    dt = prep.dtype
    for m in mod.modules():
        if id(m) in prep.m:
            continue
        if isinstance(m, L.ResnetBlock2D):
            d = {}
            d["n1"] = prep_norm(m.norm1)
            d["c1"] = prep_conv3x3(m.conv1, dt)
            d["n2"] = prep_norm(m.norm2)
            d["c2"] = prep_conv3x3(m.conv2, dt)
            d["sc"] = prep_conv1x1(m.conv_shortcut, dt) if m.conv_shortcut is not None else None
            d["temb"] = prep_linear(m.time_emb_proj, dt) if m.time_emb_proj is not None else None
            prep.put(m, d)
        elif isinstance(m, L.TemporalConvLayer):
            d = {"n": [], "c": []}
            for seq in (m.conv1, m.conv2, m.conv3, m.conv4):
                d["n"].append(prep_norm(seq[0]))
                d["c"].append(prep_conv3d_t(seq[-1], dt))
            prep.put(m, d)
        elif isinstance(m, (L.Downsample2D, L.Upsample2D)):
            prep.put(m, {"c": prep_conv3x3(m.conv, dt)})
        elif isinstance(m, L.BasicTransformerBlock):
            d = {"n1": prep_norm(m.norm1), "n3": prep_norm(m.norm3)}
            a1 = m.attn1
            d["qkv1"] = _w(torch.cat([a1.to_q.weight, a1.to_k.weight, a1.to_v.weight], dim=0), dt)
            d["o1"] = prep_linear(a1.to_out[0], dt)
            if m.attn2 is not None:
                a2 = m.attn2
                d["n2"] = prep_norm(m.norm2)
                if a2.is_cross:
                    d["q2"] = _w(a2.to_q.weight, dt)
                    d["kv2"] = _w(torch.cat([a2.to_k.weight, a2.to_v.weight], dim=0), dt)
                else:
                    d["qkv2"] = _w(torch.cat([a2.to_q.weight, a2.to_k.weight, a2.to_v.weight], dim=0), dt)
                d["o2"] = prep_linear(a2.to_out[0], dt)
            d["ff1"] = prep_linear(m.ff.net[0].proj, dt)
            d["ff2"] = prep_linear(m.ff.net[2], dt)
            prep.put(m, d)
        elif isinstance(m, (L.Transformer2DModel, L.TransformerTemporalModel)):
            prep.put(m, {"n": prep_norm(m.norm), "pi": prep_linear(m.proj_in, dt), "po": prep_linear(m.proj_out, dt)})
        elif isinstance(m, L.TimestepEmbedding):
            d = {"l1": prep_linear(m.linear_1, dt), "l2": prep_linear(m.linear_2, dt)}
            d["cp"] = _w(m.cond_proj.weight, dt) if m.cond_proj is not None else None
            prep.put(m, d)
        elif isinstance(m, L.Attention) and m.group_norm is not None:     # VAE mid-block attention
            d = {"gn": prep_norm(m.group_norm)}
            d["qkv"] = _w(torch.cat([m.to_q.weight, m.to_k.weight, m.to_v.weight], dim=0), dt)
            d["qkv_b"] = _f32(torch.cat([m.to_q.bias, m.to_k.bias, m.to_v.bias], dim=0))
            d["o"] = prep_linear(m.to_out[0], dt)
            prep.put(m, d)


# ------------------------------------------------------------------------------------------------ forward pieces
class Ctx:
    """Per-forward state shared by the blocks."""

    def __init__(self, prep: Prepared, geo: Geo):
        self.prep = prep
        self.geo = geo
        self.temb_all: Optional[torch.Tensor] = None     # fp32 [B, sum(Cout)] : time_emb_proj of every resnet
        self.temb_off: Dict[int, int] = {}               # id(resnet) -> column offset
        self.ehs: Optional[torch.Tensor] = None          # [B*Lk, 1024] 16-bit text states (one copy per batch item)
        self.lk: int = 0
        self.kv_cache: Dict[int, torch.Tensor] = {}      # id(block) -> [B*Lk, 2*inner]
        self.fuse_geglu = True
        # CFG pair with identical latents / condition / timestep: everything before the first text cross-attention is
        # computed for ONE half (batch b/2) and duplicated right there (bit-identical to computing both halves)
        self.dup_pending = False


def resnet_forward(ctx: Ctx, m: L.ResnetBlock2D, x: torch.Tensor, g: Geo, skip: Optional[torch.Tensor] = None):
    """diffusers ResnetBlock2D.forward; `skip` is the skip tensor that the reference concatenates on channels first
    (models/unet_3d_blocks.py:731,828) — here the concat is virtual."""
    p = ctx.prep.get(m)
    cin = x.shape[1] + (0 if skip is None else skip.shape[1])
    assert cin == m.in_channels
    h = ops.groupnorm(x, g.n, g.hw, p["n1"][0], p["n1"][1], m.eps, True, m.groups, x2=skip)
    bias2 = None
    if p["temb"] is not None and ctx.temb_all is not None:
        off = ctx.temb_off[id(m)]
        bias2 = ctx.temb_all[:, off: off + m.out_channels]
    # stats=True: the producing GEMM leaves per-tile column sums for the GroupNorm that reads this tensor next
    h = ops.conv3x3(h.view(g.n, g.h, g.w, cin), p["c1"][0], p["c1"][1], bias2=bias2, rows_per_bias2=g.t * g.hw, stats=True)
    h = ops.groupnorm(h, g.n, g.hw, p["n2"][0], p["n2"][1], m.eps, True, m.groups)
    if p["sc"] is not None:
        sc = ops.conv1x1_cat(x, skip, p["sc"][0], p["sc"][1])
    else:
        assert skip is None
        sc = x
    return ops.conv3x3(h.view(g.n, g.h, g.w, m.out_channels), p["c2"][0], p["c2"][1], residual=sc,
                       out_scale=1.0 / m.output_scale_factor, stats=True)


def temporal_conv_forward(ctx: Ctx, m: L.TemporalConvLayer, x: torch.Tensor, g: Geo):
    """diffusers TemporalConvLayer.forward: 4 x (GroupNorm over [b, c, t, h, w] -> SiLU -> Conv3d (3,1,1)) + identity."""
    p = ctx.prep.get(m)
    h = x
    for i in range(4):
        gn = ops.groupnorm(h, g.b, g.t * g.hw, p["n"][i][0], p["n"][i][1], 1e-5, True, 32)
        h = ops.tconv3(gn, g.b, g.t, g.hw, p["c"][i][0], p["c"][i][1], residual=x if i == 3 else None, stats=True)
    return h


def _ff(ctx: Ctx, p: dict, hs: torch.Tensor, normed: torch.Tensor):
    if ctx.fuse_geglu:
        f = ops.linear(normed, p["ff1"][0], p["ff1"][1], geglu=True)
    else:
        f = ops.geglu(ops.linear(normed, p["ff1"][0], p["ff1"][1]))
    return ops.linear(f, p["ff2"][0], p["ff2"][1], residual=hs)


def spatial_transformer_forward(ctx: Ctx, m: L.Transformer2DModel, x: torch.Tensor, g: Geo):
    """diffusers Transformer2DModel.forward (use_linear_projection=True) with BasicTransformerBlock:
    spatial self-attention over H*W tokens per frame, cross-attention to the text states, GEGLU feed-forward.
    Returns (out, g): g differs from the input geometry only when the shared CFG prefix ends here."""
    assert m.head_dim == 64, "flash kernel is specialised for head_dim 64 (the reference's attention_head_dim)"
    p = ctx.prep.get(m)
    inner = m.heads * 64
    hs = ops.groupnorm(x, g.n, g.hw, p["n"][0], p["n"][1], 1e-6, False, 32)
    hs = ops.linear(hs, p["pi"][0], p["pi"][1])
    for blk in m.transformer_blocks:
        bp = ctx.prep.get(blk)
        n1 = ops.layernorm(hs, bp["n1"][0], bp["n1"][1])
        qkv = ops.linear(n1, bp["qkv1"])
        a = ops.flash_attn_d64(qkv, 0, qkv, inner, 2 * inner, g.n, g.hw, g.hw, m.heads)
        hs = ops.linear(a, bp["o1"][0], bp["o1"][1], residual=hs)
        if blk.attn2 is not None:
            if ctx.dup_pending:
                # first use of the text states: from here on the two CFG halves differ
                hs = ops.dup_rows(hs)
                x = ops.dup_rows(x)
                g = Geo(g.b * 2, g.t, g.h, g.w)
                ctx.dup_pending = False
            n2 = ops.layernorm(hs, bp["n2"][0], bp["n2"][1])
            q = ops.linear(n2, bp["q2"])
            kv = ctx.kv_cache.get(id(blk))
            if kv is None:
                kv = ops.linear(ctx.ehs, bp["kv2"])
                ctx.kv_cache[id(blk)] = kv
            a = ops.flash_attn_d64(q, 0, kv, 0, inner, g.n, g.hw, ctx.lk, m.heads, kv_batch_div=g.t)
            hs = ops.linear(a, bp["o2"][0], bp["o2"][1], residual=hs)
        n3 = ops.layernorm(hs, bp["n3"][0], bp["n3"][1])
        hs = _ff(ctx, bp, hs, n3)
    return ops.linear(hs, p["po"][0], p["po"][1], residual=x, stats=True), g


def temporal_transformer_forward(ctx: Ctx, m: L.TransformerTemporalModel, x: torch.Tensor, g: Geo):
    """diffusers TransformerTemporalModel.forward called without encoder_hidden_states (models/unet_3d_blocks.py:379,
    526,759): GroupNorm over [b, c, t, h, w], then attention over the T frames of every pixel, twice, then GEGLU FF."""
    assert m.head_dim == 64
    p = ctx.prep.get(m)
    inner = m.heads * 64
    hs = ops.groupnorm(x, g.b, g.t * g.hw, p["n"][0], p["n"][1], 1e-6, False, 32)
    hs = ops.linear(hs, p["pi"][0], p["pi"][1])
    for blk in m.transformer_blocks:
        bp = ctx.prep.get(blk)
        for nk, qk, ok in (("n1", "qkv1", "o1"), ("n2", "qkv2", "o2")):
            if nk == "n2" and blk.attn2 is None:
                continue
            nrm = ops.layernorm(hs, bp[nk][0], bp[nk][1])
            qkv = ops.linear(nrm, bp[qk])
            a = ops.temporal_attn_d64(qkv, g.b, g.t, g.hw, m.heads, 0, inner, 2 * inner)
            hs = ops.linear(a, bp[ok][0], bp[ok][1], residual=hs)
        n3 = ops.layernorm(hs, bp["n3"][0], bp["n3"][1])
        hs = _ff(ctx, bp, hs, n3)
    return ops.linear(hs, p["po"][0], p["po"][1], residual=x, stats=True)


def downsample_forward(ctx: Ctx, m: L.Downsample2D, x: torch.Tensor, g: Geo, pad_mode="sym"):
    """Downsample2D: conv 3x3 stride 2.  Odd H / W (latent sizes that are not multiples of 8) are zero-padded to even
    first: for padding 1 the extra row / column is the conv's own zero padding, so the result is unchanged."""
    p = ctx.prep.get(m)
    x4 = x.view(g.n, g.h, g.w, m.channels)
    if (g.h | g.w) & 1:
        if pad_mode != "sym":
            raise NotImplementedError("VAE encoder needs even feature-map sizes (image height/width multiples of 8)")
        x4 = ops.pad_to_even(x4)
    out = ops.conv3x3_stride2(x4, p["c"][0], p["c"][1], pad_mode=pad_mode, stats=True)
    return out


def upsample_forward(ctx: Ctx, m: L.Upsample2D, x: torch.Tensor, g: Geo, size=None):
    """Upsample2D: nearest x2 (or to `size` = (h, w): the reference's `upsample_size` path,
    models/unet_3d_condition_mask.py:486-491) then conv 3x3."""
    p = ctx.prep.get(m)
    x4 = x.view(g.n, g.h, g.w, m.channels)
    up = ops.upsample2x(x4) if size is None or tuple(size) == (2 * g.h, 2 * g.w) else ops.upsample_nearest(x4, *size)
    return ops.conv3x3(up, p["c"][0], p["c"][1], stats=True)
