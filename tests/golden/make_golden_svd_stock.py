"""Generates `svd_stock_pipeline_tiny_ref.pt`: the stock diffusers `StableVideoDiffusionPipeline.__call__` (8-channel UNet,
no mask) pinned through the VERBATIM reference `TextStableVideoDiffusionPipeline.__call__` (models/pipeline.py:468-731)
over the diffusers shim, on the tiny SVD models of `make_golden.py`.  Run in the build container only (needs the
reference checkout, as make_golden.py does):

    python tests/golden/make_golden_svd_stock.py

With an 8-channel UNet, condition_type="image" and no condition_latent the Text call runs the stock call's ops: the image
latents (zeroed unconditional half) are the only extra input (:686-690).  Its `mask` is still concatenated for CFG (:609),
so a NaN placeholder is passed; it never reaches the UNet (the outputs are finite).  Nonzero noise_aug_strength with the
noise drawn from a fixed generator (stored as `noise`).
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import SVD_TINY, SVD_TINY_VAE, SvdImageEncoderStub, fill_deterministic  # noqa: E402  (sets sys.path)

SVD_TINY_STOCK = dict(SVD_TINY, in_channels=8)


def svd_stock_goldens():
    import diffusers                                                             # the shim
    from models.pipeline import TextStableVideoDiffusionPipeline                 # verbatim reference
    from oracle.composition import SVD_SCHED
    unet = fill_deterministic(diffusers.UNetSpatioTemporalConditionModel(**SVD_TINY_STOCK).eval(), 0)
    vae = fill_deterministic(diffusers.AutoencoderKLTemporalDecoder(**SVD_TINY_VAE).eval(), 1)
    enc = fill_deterministic(SvdImageEncoderStub().eval(), 2)
    sched = diffusers.EulerDiscreteScheduler(**SVD_SCHED)
    pipe = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=enc, unet=unet, scheduler=sched)
    g = torch.Generator().manual_seed(11)
    img = torch.randn(1, 3, 64, 128, generator=g).clamp(-1, 1)
    lat0 = torch.randn(1, 5, 4, 8, 16, generator=g)
    noise_seed = 12
    noise = torch.randn(img.shape, generator=torch.Generator().manual_seed(noise_seed))
    placeholder_mask = torch.full((1, 5, 1, 8, 16), float("nan"))                 # must not reach the UNet
    kw = dict(height=64, width=128, num_frames=5, num_inference_steps=3, decode_chunk_size=3, noise_aug_strength=0.05,
              fps=7, motion_bucket_id=100, latents=lat0, mask=placeholder_mask, return_dict=False, condition_type="image")
    out = {"unet_config": SVD_TINY_STOCK, "vae_config": SVD_TINY_VAE, "image": img, "latents_in": lat0, "noise": noise,
           "noise_seed": noise_seed, "noise_aug_strength": 0.05, "fps": 7, "motion_bucket_id": 100}
    out["latents"] = pipe(img, output_type="latent", generator=torch.Generator().manual_seed(noise_seed), **kw)
    out["frames"] = torch.stack(pipe(img, output_type="pt", generator=torch.Generator().manual_seed(noise_seed), **kw))
    torch.save(out, os.path.join(HERE, "svd_stock_pipeline_tiny_ref.pt"))
    for k in ("latents", "frames"):
        print("svd_stock_pipeline_tiny_ref.pt", k, tuple(out[k].shape), float(out[k].abs().mean()))


if __name__ == "__main__":
    svd_stock_goldens()
