"""Mirror of the reference's `utils/common.py` functions that sit on the inference path (SURVEY 8a rows a20, a22):
what `train.py:745-757` (eval) and `app.py:80` call between loading the prompt image and `pipeline.__call__`.

Same names, argument order and return values as the reference; the arithmetic runs in the sm_90a kernels
(`aab_vae_enc_finalize`, `aab_add_noise`), the random numbers come from `torch.randn` exactly as in the reference
(utils/common.py:44 / :27), so a seeded run draws the same noise.
"""
from __future__ import annotations

import torch

from . import ops


def tensor_to_vae_latent(t: torch.Tensor, vae) -> torch.Tensor:
    """utils/common.py:12-20.  t [b, f, c, h, w] in [-1, 1] -> latents [b, 4, f, h/8, w/8] = mode() * 0.18215."""
    if hasattr(vae, "encode_video_latents"):
        return vae.encode_video_latents(t, 0.18215)
    raise TypeError("tensor_to_vae_latent needs animate_anything_b200.autoencoder_kl.AutoencoderKL (no eager fallback)")


def _add_noise_16(x0: torch.Tensor, noise: torch.Tensor, alpha_prod: torch.Tensor) -> torch.Tensor:
    """sqrt(alpha_prod) * repeat(x0) + sqrt(1 - alpha_prod) * noise with torch's 16-bit scalar roundings:
    the reference computes both coefficients in the sample dtype (DDPMScheduler.add_noise casts alphas_cumprod first)."""
    a = alpha_prod.detach().to("cpu").to(noise.dtype)
    sa = float(a ** 0.5)
    sb = float((1 - a) ** 0.5)
    return ops.add_noise(x0, noise, sa, sb)


def DDPM_forward(x0: torch.Tensor, step, num_frames: int, scheduler):
    """utils/common.py:22-30: noise the repeated image latent to the scheduler's last timestep."""
    t = int(scheduler.timesteps[-1])
    shape = (x0.shape[0], x0.shape[1], num_frames, x0.shape[3], x0.shape[4])
    eps = torch.randn(shape, dtype=x0.dtype, device=x0.device)          # torch.randn_like(xt) in the reference
    alpha_vec = torch.prod(scheduler.alphas[t:])
    # the reference multiplies fp32 0-d tensors into the 16-bit latents: type promotion keeps the 16-bit dtype and casts
    # the 0-d operands to it FIRST (sqrt in fp32, then one rounding), then each product and the sum round once
    a = alpha_vec.detach().to("cpu").float()
    sa = float(torch.sqrt(a).to(x0.dtype))
    sb = float(torch.sqrt(1 - a).to(x0.dtype))
    return ops.add_noise(x0, eps, sa, sb), None


def DDPM_forward_timesteps(x0: torch.Tensor, step: int, num_frames: int, scheduler):
    """utils/common.py:32-48.  Keeps the last `step` scheduler timesteps, repeats a single-frame latent over
    `num_frames` and adds noise at the first kept timestep.  Returns (x_t [b, c, f, h, w], timesteps)."""
    timesteps = scheduler.timesteps[len(scheduler.timesteps) - step:]
    t = int(timesteps[0])
    f = num_frames if x0.shape[2] == 1 else x0.shape[2]
    shape = (x0.shape[0], x0.shape[1], f, x0.shape[3], x0.shape[4])
    noise = torch.randn(shape, dtype=x0.dtype, device=x0.device)
    return _add_noise_16(x0, noise, scheduler.alphas_cumprod[t]), timesteps


def DDPM_forward_mask(x0: torch.Tensor, step: int, num_frames: int, scheduler, mask):
    """utils/common.py:50-63: frozen region keeps the clean latent, moving region gets the noised one.
    `mask` is an HxW uint8 array / PIL image (255 = moving), resized to the latent size like the reference does."""
    import numpy as np
    import torch.nn.functional as F
    b, c, f, h, w = x0.shape
    move_xt, timesteps = DDPM_forward_timesteps(x0, step, num_frames, scheduler)
    m = torch.from_numpy(np.asarray(mask)).to(x0.device)
    if m.dim() == 2:
        m = m[None]
    else:
        m = m.permute(2, 0, 1)
    m = (m.float() / 255.0 if m.dtype == torch.uint8 else m.float()).to(x0.dtype)       # T.ToTensor()
    m = F.interpolate(m[None].float(), size=(h, w), mode="bilinear", align_corners=False, antialias=False)[0].to(x0.dtype)
    m = m[:, None, None]                                                                 # 'b h w -> b 1 1 h w'
    freeze_xt = x0.expand(-1, -1, num_frames, -1, -1) if x0.shape[2] == 1 else x0
    return freeze_xt * (1 - m) + move_xt * m, timesteps
