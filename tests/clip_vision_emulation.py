"""TEST INFRASTRUCTURE (CPU): a plain-torch restatement of diffusers 0.24's CLIP image preprocessing for PIL input (the
sequence `StableVideoDiffusionPipeline._encode_image` runs; the reference spells it out at train_svd.py:384-395), the
patch matrix `aab_clip_image_prep` writes, and stand-ins for the new `ops` wrappers (`flash_attn_d80`, `clip_image_prep`)
so that the host logic of `clip_vision.CLIPVisionModelWithProjection` can run in the CPU suite.  The restatement is pinned
to torchvision / torch / transformers by tests/test_clip_vision_cpu.py and is the oracle of the kernel in
tests/test_gpu_clip_vision.py.  The product never imports this file."""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

from animate_anything_b200 import clip_vision, ops


def gaussian_blur_reflect(x: torch.Tensor, taps_y: torch.Tensor, taps_x: torch.Tensor) -> torch.Tensor:
    """diffusers `_gaussian_blur2d`: x [B, C, H, W] fp32, the x-axis taps first, then the y-axis taps, each over a
    reflect-padded input; sums accumulated tap by tap in fp32 (the kernel's order)."""
    kx, ky = taps_x.numel(), taps_y.numel()
    px, py = (kx - 1) // 2, (ky - 1) // 2
    w = x.shape[-1]
    xp = F.pad(x, (px, kx - 1 - px, 0, 0), mode="reflect")
    bx = torch.zeros_like(x)
    for k in range(kx):
        bx = bx + taps_x[k] * xp[..., k:k + w]
    h = x.shape[-2]
    yp = F.pad(bx, (0, 0, py, ky - 1 - py), mode="reflect")
    by = torch.zeros_like(x)
    for k in range(ky):
        by = by + taps_y[k] * yp[..., k:k + h, :]
    return by


def _cubic_weights(t: torch.Tensor) -> torch.Tensor:
    """torch's bicubic weights (A = -0.75), one rounded fp32 operation at a time."""
    cc1 = lambda x: ((1.25 * x - 2.25) * x) * x + 1.0
    cc2 = lambda x: (((-0.75 * x + 3.75) * x - 6.0) * x) + 3.0
    return torch.stack([cc2(t + 1.0), cc1(t), cc1(1.0 - t), cc2(2.0 - t)], dim=-1)       # [n, 4]


def bicubic_align_corners(x: torch.Tensor, size) -> torch.Tensor:
    """Separable restatement of F.interpolate(mode="bicubic", align_corners=True) (A = -0.75, clamped borders): the
    arithmetic and summation order of the kernel, written out (x taps first, then y taps)."""
    def axis(n_in, n_out):
        f32 = lambda v: torch.tensor(float(v), dtype=torch.float32)
        scale = f32(n_in - 1) / f32(n_out - 1) if n_out > 1 else f32(0)          # fp32 division, as torch does
        real = scale * torch.arange(n_out, dtype=torch.float32)
        i0 = torch.floor(real)
        w = _cubic_weights(real - i0)
        idx = (i0.long()[:, None] + torch.arange(-1, 3)[None]).clamp(0, n_in - 1)
        return idx, w
    iy, wy = axis(x.shape[-2], size[0])
    ix, wx = axis(x.shape[-1], size[1])
    rows = torch.zeros(x.shape[:-1] + (size[1],), dtype=x.dtype)
    for l in range(4):
        rows = rows + x[..., ix[:, l]] * wx[:, l]                       # [B, C, H, Sx]
    out = torch.zeros(x.shape[:-2] + (size[0], size[1]), dtype=x.dtype)
    for k in range(4):
        out = out + rows[..., iy[:, k], :] * wy[:, k, None]
    return out


def preprocess_u8(u8: torch.Tensor, size=224, mean=clip_vision.OPENAI_CLIP_MEAN, std=clip_vision.OPENAI_CLIP_STD):
    """uint8 [B, H, W, 3] -> fp32 CLIP pixel values [B, 3, size, size], diffusers 0.24 order: /255 (pil_to_numpy),
    2x - 1, _resize_with_antialiasing, (x + 1) / 2, (x - mean) / std (CLIPImageProcessor)."""
    x = u8.permute(0, 3, 1, 2).float() / 255.0
    x = x * 2.0 - 1.0
    (ks_y, s_y), (ks_x, s_x) = clip_vision.antialias_params(x.shape[-2], x.shape[-1], (size, size))
    x = gaussian_blur_reflect(x, clip_vision.gaussian_taps(ks_y, s_y), clip_vision.gaussian_taps(ks_x, s_x))
    x = bicubic_align_corners(x, (size, size))
    x = (x + 1.0) / 2.0
    m = torch.tensor(mean, dtype=torch.float32).view(1, 3, 1, 1)
    s = torch.tensor(std, dtype=torch.float32).view(1, 3, 1, 1)
    return (x - m) / s


def patch_matrix(pixel_values: torch.Tensor, dtype, patch: int, k_pad: int) -> torch.Tensor:
    """[B, 3, S, S] -> [B * (1 + (S/patch)^2), k_pad] in `dtype`: a zero class row, then the patches (row-major grid) in the
    column order of patch_embedding.weight.flatten(1), zero columns beyond 3 patch^2."""
    b, c, s, _ = pixel_values.shape
    g = s // patch
    p = pixel_values.to(dtype).reshape(b, c, g, patch, g, patch).permute(0, 2, 4, 1, 3, 5).reshape(b, g * g, c * patch * patch)
    out = torch.zeros((b, 1 + g * g, k_pad), dtype=dtype, device=pixel_values.device)
    out[:, 1:, :c * patch * patch] = p
    return out.reshape(b * (1 + g * g), k_pad)


# ---------------------------------------------------------------------------------------------- emulated wrappers
def flash_attn_d80(q, q_col0, kv, k_col0, v_col0, nb, lq, lk, heads, kv_batch_div=1, out=None, scale=None):
    assert out is None
    scale = 1.0 / math.sqrt(80.0) if scale is None else scale
    nb_kv = kv.shape[0] // lk

    def heads_of(t, col0, n, l):
        return t[:, col0: col0 + heads * 80].float().view(n, l, heads, 80).permute(0, 2, 1, 3)
    qq = heads_of(q, q_col0, nb, lq)
    idx = torch.arange(nb) // kv_batch_div
    kk = heads_of(kv, k_col0, nb_kv, lk)[idx]
    vv = heads_of(kv, v_col0, nb_kv, lk)[idx]
    p = torch.softmax(qq @ kk.transpose(-1, -2) * scale, dim=-1)
    return (p @ vv).permute(0, 2, 1, 3).reshape(nb * lq, heads * 80)


def clip_image_prep(src, dtype, out_size, patch, k_pad, taps_y=None, taps_x=None, mean_std=None):
    if src.dtype == torch.uint8:
        ms = mean_std.tolist()
        pv = preprocess_u8(src, out_size, ms[:3], ms[3:])
    else:
        if src.shape[-2:] != (out_size, out_size):
            raise ValueError("size")
        pv = src
    return patch_matrix(pv, dtype, patch, k_pad)


@contextlib.contextmanager
def emulated_vision_ops():
    """The existing stand-ins of tests/ops_emulation.py plus the two new wrappers."""
    from ops_emulation import emulated_ops
    saved = {k: getattr(ops, k) for k in ("flash_attn_d80", "clip_image_prep")}
    try:
        with emulated_ops():
            ops.flash_attn_d80 = flash_attn_d80
            ops.clip_image_prep = clip_image_prep
            yield
    finally:
        for k, fn in saved.items():
            setattr(ops, k, fn)
