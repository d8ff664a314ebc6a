"""Generates `svd_text_batch_pipeline_tiny_ref.pt`: the VERBATIM reference `TextStableVideoDiffusionPipeline.__call__`
(models/pipeline.py:468-731) over the diffusers shim with TWO images per call (`batch_size = len(image)`, :583-588), each with
its own mask and conditioning latents, on the tiny SVD UNets of `make_golden.py` and a temporal VAE whose widths the sm_90a
mirror also takes (multiples of 64).  Run in the build container only (needs the reference checkout, as make_golden.py does):

    python tests/golden/make_golden_svd_text_batch.py

Cases (64 x 64 images, F = 5 frames, 3 Euler steps, CFG, noise augmentation from a seeded generator over the [2, 3, H, W] batch):
  condlat   9-channel UNet, the caller's `condition_latent` [2, F, 4, h, w] for both CFG halves (:631-633), decode_chunk_size = F
  image     9-channel UNet, the images' own VAE latents with zeros in the unconditional half (:624-630)
  stock8    8-channel UNet, no condition_latent, a NaN placeholder mask that never reaches the UNet (:686-690)
  straddle  as condlat with decode_chunk_size = 3: `decode_latents` chunks the flat [2 * F] frame axis, so frames 3..5 (two of
            the first video, one of the second) are decoded together and mix in the decoder's temporal layers
The decoded video is stored for `straddle` only (one file of under 1 MB).  Also stored: the exceptions the reference raises
for `num_videos_per_prompt = 2` with a mask, and for a mask of batch 1.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import SVD_TINY, SvdImageEncoderStub, fill_deterministic  # noqa: E402  (sets sys.path)

SVD_TINY_STOCK = dict(SVD_TINY, in_channels=8)
SVD_BATCH_VAE = dict(block_out_channels=(64, 64, 128, 128), layers_per_block=1)
CASES = ("condlat", "image", "stock8", "straddle")


def call_kwargs(case, gold):
    """Keyword arguments of the fixture's call for `case` (shared with the tests that replay it)."""
    kw = dict(height=64, width=64, num_frames=5, num_inference_steps=3, decode_chunk_size=3 if case == "straddle" else 5,
              noise_aug_strength=gold["noise_aug_strength"], fps=gold["fps"], motion_bucket_id=gold["motion_bucket_id"],
              latents=gold["latents_in"], return_dict=False, condition_type="image")
    kw["mask"] = torch.full_like(gold["mask"], float("nan")) if case == "stock8" else gold["mask"]
    if case in ("condlat", "straddle"):
        kw["condition_latent"] = gold["condition_latent"]
    return kw


def _error(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001  (the type is what gets recorded)
        return type(e).__name__, str(e)
    return None


def svd_text_batch_goldens():
    import diffusers                                                             # the shim
    from models.pipeline import TextStableVideoDiffusionPipeline                 # verbatim reference
    from oracle.composition import SVD_SCHED
    vae = fill_deterministic(diffusers.AutoencoderKLTemporalDecoder(**SVD_BATCH_VAE).eval(), 1)
    enc = fill_deterministic(SvdImageEncoderStub().eval(), 2)
    pipes = {}
    for ch, cfg in ((9, SVD_TINY), (8, SVD_TINY_STOCK)):
        unet = fill_deterministic(diffusers.UNetSpatioTemporalConditionModel(**cfg).eval(), 0)
        pipes[ch] = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=enc, unet=unet,
                                                     scheduler=diffusers.EulerDiscreteScheduler(**SVD_SCHED))
    g = torch.Generator().manual_seed(21)
    img = torch.randn(2, 3, 64, 64, generator=g).clamp(-1, 1)
    mask = (torch.rand(2, 5, 1, 8, 8, generator=g) > 0.5).float()
    mask[:, 0] = 0                                                               # app_svd.py:111
    lat0 = torch.randn(2, 5, 4, 8, 8, generator=g)
    cl = torch.randn(2, 5, 4, 8, 8, generator=g)
    noise_seed = 22
    out = {"unet_config": SVD_TINY, "unet_config_8ch": SVD_TINY_STOCK, "vae_config": SVD_BATCH_VAE, "image": img,
           "mask": mask, "latents_in": lat0, "condition_latent": cl, "noise_seed": noise_seed, "noise_aug_strength": 0.05,
           "fps": 7, "motion_bucket_id": 100}
    for case in CASES:
        pipe = pipes[8 if case == "stock8" else 9]
        kw = call_kwargs(case, out)
        out[f"{case}_latents"] = pipe(img, output_type="latent", generator=torch.Generator().manual_seed(noise_seed), **kw)
    # the decoded video of the straddling case only: it exercises the whole decode, and keeps the file under 1 MB
    out["straddle_frames"] = torch.stack(pipes[9](img, output_type="pt", generator=torch.Generator().manual_seed(noise_seed),
                                                  **call_kwargs("straddle", out)))
    base = call_kwargs("image", out)
    out["nvp2_error"] = _error(lambda: pipes[9](img, output_type="latent", num_videos_per_prompt=2, **base))
    out["mask_batch_error"] = _error(lambda: pipes[9](img, output_type="latent", **dict(base, mask=mask[:1])))
    torch.save(out, os.path.join(HERE, "svd_text_batch_pipeline_tiny_ref.pt"))
    for case in CASES:
        print("svd_text_batch_pipeline_tiny_ref.pt", case, tuple(out[f"{case}_latents"].shape),
              float(out[f"{case}_latents"].abs().mean()))
    print("straddle frames", tuple(out["straddle_frames"].shape), float(out["straddle_frames"].mean()))
    print("num_videos_per_prompt=2 ->", out["nvp2_error"])
    print("mask of batch 1 ->", out["mask_batch_error"])


if __name__ == "__main__":
    svd_text_batch_goldens()
