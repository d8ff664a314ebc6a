"""TEST INFRASTRUCTURE (CPU): plain-torch stand-ins for the `animate_anything_b200.ops` wrappers, with the semantics their
docstrings state (channels-last activations, tap-major conv weights, `D = act(acc + bias + bias2 + residual) * out_scale`).
They exist so that the HOST logic of a mirror class — weight-layout conversion, head padding, skip bookkeeping, geometry —
can be executed and compared with the oracle in the CPU suite, where no kernel can run.  They say nothing about the kernels
(those are compared with PyTorch references by the `-m gpu` tests) and the product never imports this file.

    with emulated_ops():
        prep = model._build_prepared(torch.float32, torch.device("cpu"))
        y = model._forward_chunk(prep, ...)
"""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

from animate_anything_b200 import ops
from animate_anything_b200._lib import ACT_GELU, ACT_NONE, ACT_QUICK_GELU, ACT_SILU


def _act(x, act):
    if act == ACT_NONE:
        return x
    if act == ACT_SILU:
        return F.silu(x)
    if act == ACT_GELU:
        return F.gelu(x)
    if act == ACT_QUICK_GELU:
        return x * torch.sigmoid(1.702 * x)
    raise ValueError(act)


def _epilogue(acc, bias=None, bias2=None, rows_per_bias2=1, residual=None, act=ACT_NONE, out_scale=1.0, out_f32=False,
              stats=False, **unused):
    bad = set(unused) - {"block_n", "direct", "ld_res", "out_rows"}
    assert not bad, bad
    if bias is not None:
        acc = acc + bias
    if bias2 is not None:
        acc = acc + bias2[torch.arange(acc.shape[0]) // rows_per_bias2]      # row / rows_per_bias2 selects the sample
    if residual is not None:
        acc = acc + residual
    return _act(acc, act) * out_scale


def linear(x, w, bias=None, geglu=False, **kw):
    acc = x.float() @ w.float().t()
    if geglu:
        nh = acc.shape[1] // 2
        b = 0 if bias is None else bias
        acc = acc + b
        return acc[:, :nh] * F.gelu(acc[:, nh:])
    return _epilogue(acc, bias, **kw)


def conv1x1_cat(x, x2, w, bias=None, **kw):
    return linear(x if x2 is None else torch.cat([x, x2], dim=1), w, bias, **kw)


def _w4(w, cin):
    co = w.shape[0]
    return w.float().view(co, 3, 3, cin).permute(0, 3, 1, 2)


def conv3x3(x, w, bias=None, x2=None, **kw):
    if x2 is not None:
        x = torch.cat([x, x2], dim=-1)
    n, h, wd, c = x.shape
    y = F.conv2d(x.float().permute(0, 3, 1, 2), _w4(w, c), padding=1)
    return _epilogue(y.permute(0, 2, 3, 1).reshape(n * h * wd, -1), bias, **kw)


def conv3x3_stride2(x, w, bias=None, pad_mode="sym", **kw):
    n, h, wd, c = x.shape
    assert h % 2 == 0 and wd % 2 == 0 and c % 64 == 0          # the wrapper's own assertion
    xi = x.float().permute(0, 3, 1, 2)
    if pad_mode == "sym":
        y = F.conv2d(xi, _w4(w, c), stride=2, padding=1)
    else:
        y = F.conv2d(F.pad(xi, (0, 1, 0, 1)), _w4(w, c), stride=2)
    return _epilogue(y.permute(0, 2, 3, 1).reshape(-1, y.shape[1]), bias, **kw)


def groupnorm(x, samples, rows, gamma, beta, eps, silu, groups=32, x2=None):
    if x2 is not None:
        x = torch.cat([x, x2], dim=1)
    c = x.shape[1]
    assert x.shape[0] == samples * rows and c % groups == 0
    v = x.float().view(samples, rows, groups, c // groups)
    mean = v.mean(dim=(1, 3), keepdim=True)
    var = v.var(dim=(1, 3), keepdim=True, unbiased=False)
    y = ((v - mean) / torch.sqrt(var + eps)).view(samples * rows, c) * gamma + beta
    return F.silu(y) if silu else y


def flash_attn_d64(q, q_col0, kv, k_col0, v_col0, nb, lq, lk, heads, kv_batch_div=1, out=None, causal=False, scale=None):
    assert not causal and out is None
    scale = 1.0 / math.sqrt(64.0) if scale is None else scale
    nb_kv = kv.shape[0] // lk

    def heads_of(t, col0, n, l):
        return t[:, col0: col0 + heads * 64].float().view(n, l, heads, 64).permute(0, 2, 1, 3)
    qq = heads_of(q, q_col0, nb, lq)
    idx = torch.arange(nb) // kv_batch_div
    kk = heads_of(kv, k_col0, nb_kv, lk)[idx]
    vv = heads_of(kv, v_col0, nb_kv, lk)[idx]
    p = torch.softmax(qq @ kk.transpose(-1, -2) * scale, dim=-1)
    return (p @ vv).permute(0, 2, 1, 3).reshape(nb * lq, heads * 64)


def image_to_nhwc8(img):
    n, c, h, w = img.shape
    out = torch.zeros((n, h, w, 8), dtype=img.dtype)
    out[..., :c] = img.permute(0, 2, 3, 1)
    return out


def video_f32_to_nhwc8(video, dtype):
    b, c, f, h, w = video.shape
    out = torch.zeros((b * f, h, w, 8), dtype=dtype)
    out[..., :c] = video.permute(0, 2, 3, 4, 1).reshape(b * f, h, w, c).to(dtype)
    return out


def upsample2x(x):
    return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)


def pad_cols(x, dst_cols):
    assert x.shape[1] % 8 == 0 and dst_cols % 8 == 0
    return F.pad(x, (0, dst_cols - x.shape[1]))


def cat_cols(x, x2):
    return torch.cat([x, x2], dim=1)


def svd_out_finalize(y, b, f, h, w, dtype):
    return y[:, :4].reshape(b, f, h, w, 4).permute(0, 1, 4, 2, 3).to(dtype)


def rgba_finalize_u8(y, pixels, bf16):
    dt = torch.bfloat16 if bf16 else torch.float16
    v = y[:pixels, :4].to(dt)
    fg = ((v[:, :3] + 1.0) * 127.5).float().clamp(0, 255)
    a = v[:, 3:] * 255.0
    a = torch.where(a > 127, torch.full_like(a, 255.0), torch.zeros_like(a)).float()
    return torch.cat([fg, a], dim=1).to(torch.uint8)


# ---------------------------------------------------------------------------------------------- main UNet3D path
def unet_in_assemble(sample, cond, mask, t_frames):
    """[B,4,F,h,w] + [B,4,1,h,w] (+ mask [Bm,1,1,h,w], batch b reads mask b % Bm) -> [B, T, h, w, 8], channels (mask, c0..c3, 0...)."""
    b, _, f, h, w = sample.shape
    x = torch.cat([cond, sample], dim=2).permute(0, 2, 3, 4, 1)            # [B, T, h, w, 4]
    out = torch.zeros((b, f + 1, h, w, 8), dtype=sample.dtype)
    if mask is not None:
        idx = torch.arange(b) % mask.shape[0]
        out[..., 0] = mask[idx, 0, 0][:, None].expand(b, f + 1, h, w)
        out[..., 1:5] = x
    else:
        out[..., :4] = x
    return out


def unet_out_finalize(y, b, t, h, w, dtype):
    return y[:, :4].reshape(b, t, h, w, 4)[:, 1:].permute(0, 4, 1, 2, 3).to(dtype).contiguous()


def timestep_embed(t, b, dim, dtype):
    half = dim // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    tv = t.float().reshape(-1)[torch.arange(b) % t.numel()]
    a = tv[:, None] * freq[None]
    return torch.cat([torch.cos(a), torch.sin(a)], dim=1).to(dtype)


def layernorm(x, gamma, beta, eps=1e-5):
    return F.layer_norm(x.float(), (x.shape[1],), gamma, beta, eps)


def temporal_attn_d64(qkv, b, t, hw, heads, q_col0, k_col0, v_col0):
    """rows ordered (b, t, hw); attention over t for every (b, pixel, head)."""
    def pick(col0):
        return qkv[:, col0: col0 + heads * 64].float().view(b, t, hw, heads, 64).permute(0, 2, 3, 1, 4)   # b hw heads t 64
    q, k, v = pick(q_col0), pick(k_col0), pick(v_col0)
    p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(64.0), dim=-1)
    return (p @ v).permute(0, 3, 1, 2, 4).reshape(b * t * hw, heads * 64)


def tconv3(x, b, t, hw, w, bias=None, **kw):
    c = x.shape[1]
    xi = x.float().view(b, t, hw, c).permute(0, 3, 1, 2)                   # b c t hw
    w5 = w.float().view(w.shape[0], 3, c).permute(0, 2, 1)[..., None]      # [Cout, C, 3, 1]
    y = F.conv2d(xi, w5, padding=(1, 0))
    return _epilogue(y.permute(0, 2, 3, 1).reshape(b * t * hw, -1), bias, **kw)


def dup_rows(x):
    return torch.cat([x, x], dim=0)


def geglu(x):
    nh = x.shape[1] // 2
    return x[:, :nh] * F.gelu(x[:, nh:].float())


def upsample_nearest(x, oh, ow):
    return F.interpolate(x.float().permute(0, 3, 1, 2), size=(oh, ow), mode="nearest").permute(0, 2, 3, 1).contiguous()


def pad_to_even(x):
    n, h, w, c = x.shape
    return F.pad(x, (0, 0, 0, w & 1, 0, h & 1))


def cfg_scheduler_step(eps, ldc, cfg, guidance, x, x_out, x0_hist, coef, step_idx):
    """eps fp32 [Bu*T*h*w, >=4] channels-last with T = F + 1 (frame 0 = the condition frame, dropped), CFG halves ordered
    [uncond..., text...]; x, x_out [n, 4, F, h, w]; coef one row of 6 (or a table indexed by step_idx)."""
    n, _, f, h, w = x.shape
    k = (coef if step_idx is None else coef[int(step_idx)]).reshape(-1)[:6].double()
    e = eps[:, :4].double().reshape(-1, f + 1, h, w, 4)[:, 1:].permute(0, 4, 1, 2, 3)      # [Bu, 4, F, h, w]
    if cfg:
        e = e[:n] + guidance * (e[n:] - e[:n])
    xv = x.double()
    x0 = k[0] * xv + k[1] * e
    xn = k[2] * xv + k[3] * e + k[4] * x0
    if x0_hist is not None:
        xn = xn + k[5] * x0_hist.double()
        x0_hist.copy_(x0.to(x0_hist.dtype))
    x_out.copy_(xn.to(x_out.dtype))
    return x_out


# ---------------------------------------------------------------------------------------------- SD VAE path
def igemm(a, a_dims, a_strides, w, n, kc, dim_d, box, taps, out=None, ld_out=None, *, b_batch=0, b_batch_stride=0, b_batch_dim=-1,
          ld_b=None, **kw):
    """Only the form AutoencoderKL._mid_attention uses: no taps, A a 2-D [rows, >= kc] matrix, B batched over output dim 1
    (`b_batch` matrices of `n` rows x `kc` columns, `b_batch_stride` elements apart inside `w`'s storage)."""
    assert len(taps) == 1 and not any(taps[0]) and b_batch >= 1 and b_batch_dim == 1 and out is None
    rows_per = dim_d[0]
    a2 = a.float()[:, :kc]
    ld = ld_b if ld_b is not None else w.stride(-2)
    outs = []
    for b in range(b_batch):
        wb = torch.as_strided(w, (n, kc), (ld, 1), w.storage_offset() + b * b_batch_stride).float()
        outs.append(a2[b * rows_per:(b + 1) * rows_per] @ wb.t())
    return _epilogue(torch.cat(outs, dim=0), **kw)


def softmax_rows(s, dtype, pad_to=None):
    p = torch.softmax(s.float(), dim=1).to(dtype)
    return p if not pad_to or pad_to == p.shape[1] else F.pad(p, (0, pad_to - p.shape[1]))


def transpose_batched(src, col0, nb, rows, cols, ld=None):
    ld = ld or rows
    dst = torch.zeros((nb, cols, ld), dtype=src.dtype)
    dst[:, :, :rows] = src[:, col0: col0 + cols].reshape(nb, rows, cols).permute(0, 2, 1)
    return dst


def vae_enc_finalize(mom, wq, bq, scale, b, f, h, w):
    m = mom[:, :8].float() @ wq.float().t() + bq                                    # quant_conv 1x1
    return (m * scale).reshape(b, f, h, w, 8).permute(0, 4, 1, 2, 3).to(mom.dtype).contiguous()


def vae_dec_in(lat, inv_scale, wp, bp):
    b, _, f, h, w = lat.shape
    z = (lat.float() * inv_scale).permute(0, 2, 3, 4, 1).reshape(-1, 4) @ wp.float().t() + bp     # post_quant_conv 1x1
    out = torch.zeros((b * f, h, w, 8), dtype=lat.dtype)
    out[..., :4] = z.reshape(b * f, h, w, 4).to(lat.dtype)
    return out


def vae_dec_finalize(y, b, f, h, w, bf16):
    return y[:, :3].float().reshape(b, f, h, w, 3).permute(0, 4, 1, 2, 3).contiguous()


def vae_dec_finalize_u8(y, b, f, h, w, bf16):
    v = y[:, :3].float().reshape(b, f, h, w, 3)
    v = ((v * 0.5 + 0.5).clamp(0, 1) * 255).to(torch.uint8)
    return v.permute(1, 2, 0, 3, 4).reshape(f, h, b * w, 3).contiguous()


# ---------------------------------------------------------------------------------------------- SVD path
def image_to_nhwc16(img):
    n, c, h, w = img.shape
    out = torch.zeros((n, h, w, 16), dtype=img.dtype)
    out[..., :c] = img.permute(0, 2, 3, 1)
    return out


def add_rowvec(x, vec, rows_per_vec, mod, mode=0, mod2=1, inplace=False):
    """x[r] + vec[idx(r)]; mode 0: idx = (r // rows_per_vec) % mod; mode 1 (rows (b, f, s), S = rows_per_vec, F = mod2):
    idx = (b * S + s) % mod."""
    r = torch.arange(x.shape[0])
    if mode == 0:
        idx = (r // rows_per_vec) % mod
    else:
        s_ = r % rows_per_vec
        b_ = r // (rows_per_vec * mod2)
        idx = (b_ * rows_per_vec + s_) % mod
    out = x + vec.to(x.dtype)[idx]
    if inplace:
        x.copy_(out)
        return x
    return out


def axpby(x, y, a, b):
    return a * x + b * y


def svd_in_assemble_frames(x, cond, mask, sigma, cfg, zero_uncond):
    """x [B, F, 4, h, w]; cond [Hc, B, F' in (1, F), 4, h, w]; mask [B, F, h, w] or None -> [(2)B*F, h, w, 16]:
    channels (mask?, x / sqrt(sigma^2 + 1), cond); the unconditional half (first) sees zero cond when `zero_uncond`."""
    b, f, _, h, w = x.shape
    xs = (x / math.sqrt(sigma * sigma + 1.0)).reshape(b * f, 4, h, w)
    halves = []
    for half in ((0, 1) if cfg else (1,)):
        c = cond[min(half, cond.shape[0] - 1)] if cfg else cond[cond.shape[0] - 1]
        c = c.expand(b, f, 4, h, w).reshape(b * f, 4, h, w)
        if half == 0 and zero_uncond:
            c = torch.zeros_like(c)
        parts = ([mask.reshape(b * f, 1, h, w)] if mask is not None else []) + [xs, c]
        halves.append(torch.cat(parts, dim=1))
    return image_to_nhwc16(torch.cat(halves, dim=0))


def svd_in_assemble(x, img_lat, mask, sigma, cfg):
    b, f, _, h, w = x.shape
    return svd_in_assemble_frames(x, img_lat.reshape(1, b, 1, 4, h, w), mask.reshape(1, 1, h, w).expand(b, f, h, w), sigma, cfg, True)


def svd_cfg_euler_step(pred, cfg, gs, x, sigma, sigma_next):
    b, f, _, h, w = x.shape
    p = pred[:, :4].float().reshape(-1, f, h, w, 4).permute(0, 1, 4, 2, 3)                 # [(2)B, F, 4, h, w]
    v = p[:b] + gs.float().reshape(1, f, 1, 1, 1) * (p[b:] - p[:b]) if cfg else p
    xs = x.float()
    s2 = sigma * sigma + 1.0
    x0 = v * (-sigma / math.sqrt(s2)) + xs / s2
    return (xs + (xs - x0) / sigma * (sigma_next - sigma)).to(x.dtype)


_EMULATED = dict(svd_in_assemble=svd_in_assemble, svd_in_assemble_frames=svd_in_assemble_frames,
                 svd_cfg_euler_step=svd_cfg_euler_step, image_to_nhwc16=image_to_nhwc16, add_rowvec=add_rowvec, axpby=axpby, igemm=igemm, softmax_rows=softmax_rows, transpose_batched=transpose_batched, vae_enc_finalize=vae_enc_finalize,
                 vae_dec_in=vae_dec_in, vae_dec_finalize=vae_dec_finalize, vae_dec_finalize_u8=vae_dec_finalize_u8,
                 cfg_scheduler_step=cfg_scheduler_step, unet_in_assemble=unet_in_assemble, unet_out_finalize=unet_out_finalize, timestep_embed=timestep_embed,
                 layernorm=layernorm, temporal_attn_d64=temporal_attn_d64, tconv3=tconv3, dup_rows=dup_rows, geglu=geglu,
                 upsample_nearest=upsample_nearest, pad_to_even=pad_to_even, linear=linear, conv1x1_cat=conv1x1_cat, conv3x3=conv3x3, conv3x3_stride2=conv3x3_stride2, groupnorm=groupnorm,
                 flash_attn_d64=flash_attn_d64, image_to_nhwc8=image_to_nhwc8, video_f32_to_nhwc8=video_f32_to_nhwc8,
                 upsample2x=upsample2x, pad_cols=pad_cols, cat_cols=cat_cols, svd_out_finalize=svd_out_finalize,
                 rgba_finalize_u8=rgba_finalize_u8)


@contextlib.contextmanager
def emulated_ops():
    saved = {k: getattr(ops, k) for k in _EMULATED}
    try:
        for k, fn in _EMULATED.items():
            setattr(ops, k, fn)
        yield
    finally:
        for k, fn in saved.items():
            setattr(ops, k, fn)
