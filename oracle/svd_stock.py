"""ORACLE (test infrastructure, not product): plain-PyTorch restatement of diffusers 0.24
`StableVideoDiffusionPipeline.__call__` (the stock image-to-video call with an 8-channel UNet, no mask), on the same
diffusers shim as `oracle/composition.py`.

  oracle_svd_stock_sampling_loop  <- the loop of models/pipeline.py:375-459 without the mask (:373 dropped, :422 reduced
                                     to cat([latent_model_input, image_latents], dim=2))

Pinned to the verbatim `TextStableVideoDiffusionPipeline.__call__` (models/pipeline.py:468-731) with an 8-channel UNet,
condition_type="image" and no condition_latent, which computes the same ops: its mask is concatenated for CFG (:609) but
an 8-channel input never reads it (:686-690).  The fixture is `tests/golden/svd_stock_pipeline_tiny_ref.pt`, written by
`tests/golden/make_golden_svd_stock.py` and checked by `tests/test_svd_stock_cpu.py`.
"""
from __future__ import annotations

import torch

from oracle.composition import AutoencoderKLTemporalDecoder, EulerDiscreteScheduler, SVD_SCHED  # noqa: F401


@torch.no_grad()
def oracle_svd_stock_sampling_loop(unet, scheduler, vae, image_embeddings, image_latents, latents, num_inference_steps=25,
                                   min_guidance_scale=1.0, max_guidance_scale=3.0, fps=6, motion_bucket_id=127,
                                   noise_aug_strength=0.02, decode_chunk_size=None, decode=True):
    """From the point where the image has been encoded: `image_embeddings` [B, 1, D] (positive half), `image_latents`
    [B, 4, h, w] (`vae.encode(image + noise_aug_strength * noise).latent_dist.mode()`, not scaled), `latents`
    [B, F, 4, h, w] unit noise, `fps` already reduced by one.  Classifier-free guidance with zeroed negative conditioning,
    per-frame guidance scale linspace(min, max, F), 8-channel input cat([x, image_latents], dim=2), Euler steps, chunked
    temporal-VAE decode.  Returns (frames [B, 3, F, H, W] fp32 or None, latents)."""
    b, nf = latents.shape[:2]
    cfg = max_guidance_scale > 1.0
    emb = torch.cat([torch.zeros_like(image_embeddings), image_embeddings]) if cfg else image_embeddings
    il = torch.cat([torch.zeros_like(image_latents), image_latents]) if cfg else image_latents
    il = il.unsqueeze(1).repeat(1, nf, 1, 1, 1)
    ids = torch.tensor([[fps, motion_bucket_id, noise_aug_strength]], dtype=emb.dtype).repeat(b, 1)
    ids = (torch.cat([ids, ids]) if cfg else ids).to(latents.device)
    scheduler.set_timesteps(num_inference_steps, device=latents.device)
    latents = latents * scheduler.init_noise_sigma
    gs = torch.linspace(min_guidance_scale, max_guidance_scale, nf).unsqueeze(0).to(latents.device, latents.dtype)
    gs = gs.repeat(b, 1)[:, :, None, None, None]
    for t in scheduler.timesteps:
        x = torch.cat([latents] * 2) if cfg else latents
        x = scheduler.scale_model_input(x, t)
        x = torch.cat([x, il], dim=2)
        pred = unet(x, t, encoder_hidden_states=emb, added_time_ids=ids, return_dict=False)[0]
        if cfg:
            pu, pc = pred.chunk(2)
            pred = pu + gs * (pc - pu)
        latents = scheduler.step(pred, t, latents).prev_sample
    if not decode:
        return None, latents
    chunk = decode_chunk_size or nf
    z = latents.flatten(0, 1) / vae.config.scaling_factor
    frames = torch.cat([vae.decode(z[i: i + chunk], num_frames=z[i: i + chunk].shape[0]).sample
                        for i in range(0, z.shape[0], chunk)], dim=0)
    frames = frames.reshape(-1, nf, *frames.shape[1:]).permute(0, 2, 1, 3, 4).float()
    return frames, latents
