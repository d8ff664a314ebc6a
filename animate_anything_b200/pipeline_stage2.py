"""Mirror of the reference's `models/pipeline_stage2.py` `MaskedLatentToVideoPipeline.__call__` (:171-337), the
transparent-video (RGBA) generation call of `train_transparent_i2v_stage2.py:500-515` (SURVEY row f4).

Relation to the main path: the denoising loop (:252-296) is `LatentToVideoPipeline.__call__`'s loop (models/pipeline.py:
156-197) token for token — `encode_prompt` returns the (positive, negative) tuple which :232 re-concatenates as
[negative, positive], the condition latent is duplicated for the guidance halves (:249-250), same UNet keywords, same CFG
combine and scheduler step — so it runs through the same captured-graph step.  What this class adds is the tail
(:299-324): `decode_latents`, then the `UNet384` alpha decoder on (decoded frames, final latents) and the RGBA
post-processing, here `vae_alpha_decoder.decode_rgba_u8` (layerdiffuse_VAE.py): one pass from the fp32 video to uint8
RGBA frames on the device.

Called unbound on a base pipeline object, exactly like the reference does (`MaskedLatentToVideoPipeline.__call__(pipeline,
...)` with `pipeline = TextToVideoSDPipeline.from_pretrained(...)`, train_transparent_i2v_stage2.py:565): `self` only
needs the attributes of `LatentToVideoPipeline`, which is what `TextToVideoSDPipeline` is bound to here.

Deviation, stated: the reference passes `image_embeds=image_embeds` to the UNet unconditionally (:282), a keyword that
`models/unet_3d_condition_mask.py:338-353` does not accept — as written the call raises TypeError with the repository's own
UNet (recorded in tests/golden/transparent_ref.pt).  The mirror does not forward the keyword (the trainer leaves it at None);
a non-None value raises NotImplementedError.
`ImageToVideoPipeline` (:11-169, an `_encode_prompt` variant with image embeddings) and `ConcatLatentToVideoPipeline`
(:339-590, an 8-channel UNet called without `condition_latent`) drive UNet variants that are not in the reference tree and
are not mirrored.
"""
from __future__ import annotations

import torch

from .pipeline import LatentToVideoPipeline, TextToVideoSDPipelineOutput

TextToVideoSDPipeline = LatentToVideoPipeline      # the binding for `from diffusers import TextToVideoSDPipeline` (:5)


class MaskedLatentToVideoPipeline(LatentToVideoPipeline):
    @torch.no_grad()
    def __call__(self, clean_latents=None, vae_alpha_decoder=None, prompt=None, height=None, width=None,
                 num_frames: int = 16, num_inference_steps: int = 50, guidance_scale=9.0, negative_prompt=None,
                 eta: float = 0.0, generator=None, latents=None, condition_latent=None, prompt_embeds=None,
                 negative_prompt_embeds=None, output_type="np", return_dict: bool = True, callback=None,
                 callback_steps: int = 1, cross_attention_kwargs=None, timesteps=None, mask=None, motion=None,
                 image_embeds=None):
        from . import _lib
        launches0 = _lib.launch_count()
        if image_embeds is not None:
            raise NotImplementedError("image_embeds: models/unet_3d_condition_mask.py:338-353 has no such argument "
                                      "(the reference's own call at models/pipeline_stage2.py:282 raises TypeError)")
        if vae_alpha_decoder is None:
            raise TypeError("'NoneType' object is not callable")       # what :308 raises without a decoder
        if not hasattr(vae_alpha_decoder, "decode_rgba_u8"):
            raise TypeError("vae_alpha_decoder must be animate_anything_b200.layerdiffuse_VAE.UNet384 (the sm_90a mirror of "
                            "models/layerdiffuse_VAE.py:UNet384); a torch module would mean an eager fallback, which this "
                            "path does not have")
        _, latents = LatentToVideoPipeline.__call__(
            self, prompt=prompt, height=height, width=width, num_frames=num_frames,
            num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, negative_prompt=negative_prompt, eta=eta,
            generator=generator, latents=latents, prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
            output_type="latent", return_dict=False, callback=callback, callback_steps=callback_steps,
            cross_attention_kwargs=cross_attention_kwargs, condition_latent=condition_latent, mask=mask, timesteps=timesteps,
            motion=motion)
        # decode_latents (:299): fp32 [b, 3, f, H, W]; the tensor2vid frames (:330) come from the same decoder pass
        video_tensor, frames_u8 = self.vae.decode_video_and_frames_uint8(latents)
        b = video_tensor.shape[0]
        pngs_dev = vae_alpha_decoder.decode_rgba_u8(video_tensor, latents)      # :303-324 fused, uint8 [f, H, W, 4]
        pngs = pngs_dev.cpu().numpy()
        pngs_rgb = pngs[:, :, :, :3]
        alpha_jpg = pngs[:, :, :, 3]
        assert b == 1                                                  # :327
        if output_type == "pt":
            video = video_tensor
        else:
            frames = frames_u8.cpu().numpy()
            video = [frames[i] for i in range(frames.shape[0])]
        self.last_gpu_launches = _lib.launch_count() - launches0
        if not return_dict:
            return (video, latents, pngs, alpha_jpg, pngs_rgb)
        return TextToVideoSDPipelineOutput(frames=video)
