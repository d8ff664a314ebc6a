"""Mirror of the reference's `MaskStableVideoDiffusionPipeline.__call__` (models/pipeline.py:223-466; BASELINE config
4, driven by train_svd.py:756-777): same keyword arguments, defaults and return values.

What is mirrored on the sm_90a kernels (the hot path, reference line -> here):
  :359-362  `_encode_vae_image` (VAE encode of the noise-augmented image, `latent_dist.mode()`)  -> AutoencoderKLTemporalDecoder.encode
  :418-422  `cat([latents] * 2)`, `scale_model_input`, `cat([mask, x, image_latents], dim=2)`       -> ONE kernel, `aab_svd_in_assemble`
  :425-431  UNetSpatioTemporalConditionModel.forward                                              -> unet_spatio_temporal_condition.py
  :434-439  per-frame guidance (`linspace(min, max, F)`, :405-408) + EulerDiscreteScheduler.step  -> ONE kernel, `aab_svd_cfg_euler_step`
  :456      `decode_latents` in chunks of `decode_chunk_size` frames                                -> decode_chunk_video
What stays a library call: the CLIP *vision* tower of `_encode_image` (:343; once per clip, outside SURVEY.md 8's rows) — any
module mapping the image batch to embeddings (`.image_embeds` or a tensor) is accepted, or pass `image_embeddings=`.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Union

import torch

from . import ops
from .modeling import BaseOutput


class StableVideoDiffusionPipelineOutput(BaseOutput):
    pass


def _append_dims(x, target_dims):
    """models/pipeline.py:216-221."""
    dims_to_append = target_dims - x.ndim
    if dims_to_append < 0:
        raise ValueError(f"input has {x.ndim} dims but target_dims is {target_dims}, which is less")
    return x[(...,) + (None,) * dims_to_append]


class MaskStableVideoDiffusionPipeline:
    def __init__(self, vae, image_encoder, unet, scheduler, feature_extractor=None):
        self.vae, self.image_encoder, self.unet, self.scheduler = vae, image_encoder, unet, scheduler
        self.feature_extractor = feature_extractor
        self.vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
        from .image_processor import VaeImageProcessor
        self.image_processor = VaeImageProcessor(vae_scale_factor=self.vae_scale_factor)
        self.last_gpu_launches = 0

    @property
    def guidance_scale(self):
        return self._guidance_scale

    def check_inputs(self, image, height, width):
        import PIL.Image
        if not isinstance(image, torch.Tensor) and not isinstance(image, PIL.Image.Image) and not isinstance(image, list):
            raise ValueError("`image` has to be of type `torch.FloatTensor` or `PIL.Image.Image` or `List[PIL.Image.Image]` but is"
                             f" {type(image)}")
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")

    def _encode_image(self, image, device, num_videos_per_prompt, do_classifier_free_guidance):
        """CLIP image embedding [B, 1, D]; under CFG returns cat([zeros, embeddings]) (diffusers _encode_image)."""
        dtype = self.unet.dtype
        out = self.image_encoder(image.to(device=device, dtype=next(self.image_encoder.parameters()).dtype))
        emb = out.image_embeds if hasattr(out, "image_embeds") else out
        emb = emb.to(dtype).unsqueeze(1)
        bs, seq, _ = emb.shape
        emb = emb.repeat(1, num_videos_per_prompt, 1).view(bs * num_videos_per_prompt, seq, -1)
        if do_classifier_free_guidance:
            emb = torch.cat([torch.zeros_like(emb), emb])
        return emb

    def decode_latents(self, latents, num_frames, decode_chunk_size=14):
        """diffusers StableVideoDiffusionPipeline.decode_latents: [B, F, 4, h, w] -> fp32 [B, 3, F, H, W], decoded in
        chunks of `decode_chunk_size` frames (the temporal layers of the decoder see one chunk at a time)."""
        lat = latents.flatten(0, 1)
        if latents.shape[0] != 1:
            raise NotImplementedError("one video per call (as the reference's mask handling implies, models/pipeline.py:372)")
        outs = []
        inv = 1.0 / self.vae.config.scaling_factor
        for i in range(0, lat.shape[0], decode_chunk_size):
            z = lat[i: i + decode_chunk_size]
            # 1 / scaling_factor * latents: python float times 16-bit tensor -> one rounding (done by torch here: a scalar
            # scale of a [n, 4, h, w] latent, once per clip)
            z = (z * inv).contiguous()
            outs.append(self.vae.decode_chunk_video(z, z.shape[0]))           # [1, 3, n, H, W] fp32
        return torch.cat(outs, dim=2)                                         # [1, 3, F, H, W]: chunks are consecutive frames

    @torch.no_grad()
    def __call__(self, image, height: int = 576, width: int = 1024, num_frames: Optional[int] = None,
                 num_inference_steps: int = 25, min_guidance_scale: float = 1.0, max_guidance_scale: float = 3.0,
                 fps: int = 7, motion_bucket_id: int = 127, noise_aug_strength: float = 0.02,
                 decode_chunk_size: Optional[int] = None, num_videos_per_prompt: Optional[int] = 1,
                 generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
                 latents: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 callback_on_step_end: Optional[Callable[[int, int, Dict], None]] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"], return_dict: bool = True, mask=None,
                 image_embeddings: Optional[torch.Tensor] = None):
        from . import _lib
        launches0 = _lib.launch_count()
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        num_frames = num_frames if num_frames is not None else self.unet.config.num_frames
        decode_chunk_size = decode_chunk_size if decode_chunk_size is not None else num_frames
        self.check_inputs(image, height, width)
        if mask is None:
            raise ValueError("MaskStableVideoDiffusionPipeline needs `mask` ([1, h/8, w/8]; models/pipeline.py:372)")
        device = self.unet.device
        dtype = self.unet.dtype
        cfg = max_guidance_scale > 1.0
        # 3. image embedding (library call, once per clip) unless supplied
        image_t = self.image_processor.preprocess(image, height=height, width=width).to(device)
        batch_size = image_t.shape[0]
        if batch_size * num_videos_per_prompt != 1:
            raise NotImplementedError("the reference's mask handling ('1 h w -> 2 f 1 h w', :372) implies one video per call")
        if image_embeddings is None:
            image_embeddings = self._encode_image(image_t, device, num_videos_per_prompt, cfg)
        else:
            image_embeddings = image_embeddings.to(device=device, dtype=dtype)
            if cfg and image_embeddings.shape[0] == batch_size:
                image_embeddings = torch.cat([torch.zeros_like(image_embeddings), image_embeddings])
        fps = fps - 1
        # 4. VAE-encode the noise-augmented image (:352-362); needs_upcasting (:355) is moot: the sm_90a path is 16-bit
        noise = torch.randn(image_t.shape, generator=generator, device=generator.device if generator is not None else device,
                            dtype=image_t.dtype).to(device)
        image_t = image_t + noise_aug_strength * noise
        image_latents = self.vae.encode(image_t.to(dtype)).latent_dist.mode().to(dtype).contiguous()     # [1, 4, h, w]
        # 5. added time ids (_get_add_time_ids)
        ids = torch.tensor([[fps, motion_bucket_id, noise_aug_strength]], dtype=dtype).repeat(batch_size, 1)
        ids = (torch.cat([ids, ids]) if cfg else ids).to(device)
        # 4'. timesteps / sigmas
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        timesteps = self.scheduler.timesteps
        sigmas = [float(s) for s in self.scheduler.sigmas]
        # 5'. latents (prepare_latents)
        c_lat = self.unet.config.in_channels // 2
        shape = (batch_size, num_frames, c_lat, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if latents is None:
            latents = torch.randn(shape, generator=generator, device=generator.device if generator is not None else device,
                                  dtype=dtype).to(device)
        else:
            latents = latents.to(device=device, dtype=dtype)
        latents = (latents * float(self.scheduler.init_noise_sigma)).contiguous()
        # 7. per-frame guidance scale (:405-408)
        gs = torch.linspace(min_guidance_scale, max_guidance_scale, num_frames).unsqueeze(0).to(device, latents.dtype)
        self._guidance_scale = _append_dims(gs.repeat(batch_size, 1), latents.ndim)
        gs_f32 = gs[0].float().contiguous()
        m16 = mask.to(device=device, dtype=dtype).reshape(shape[3], shape[4]).contiguous()
        in_ch = self.unet.config.in_channels
        b_unet = (2 if cfg else 1) * batch_size
        # 8. denoising loop
        self._num_timesteps = len(timesteps)
        for i, t in enumerate(timesteps):
            x16 = ops.svd_in_assemble(latents, image_latents, m16, sigmas[i], cfg)
            pred, _ = self.unet(None, t, image_embeddings, ids, _raw=True, _x16=x16,
                                _shape=(b_unet, num_frames, in_ch, shape[3], shape[4]))
            latents = ops.svd_cfg_euler_step(pred, cfg, gs_f32, latents, sigmas[i], sigmas[i + 1])
            if callback_on_step_end is not None:
                callback_kwargs = {k: locals()[k] for k in callback_on_step_end_tensor_inputs}
                callback_outputs = callback_on_step_end(self, i, t, callback_kwargs)
                latents = callback_outputs.pop("latents", latents)
        if output_type != "latent":
            frames = self.decode_latents(latents, num_frames, decode_chunk_size)
            frames = [self.image_processor.postprocess(frames[b].permute(1, 0, 2, 3), output_type)
                      for b in range(frames.shape[0])]                       # diffusers svd tensor2vid
        else:
            frames = latents
        self.last_gpu_launches = _lib.launch_count() - launches0
        if not return_dict:
            return frames
        return StableVideoDiffusionPipelineOutput(frames=frames)


class TextStableVideoDiffusionPipeline(MaskStableVideoDiffusionPipeline):
    """Mirror of the reference's `TextStableVideoDiffusionPipeline.__call__` (models/pipeline.py:468-731): the SVD loop
    conditioned on the CLIP image embedding (`condition_type="image"`), on text embeddings (`"text"`: prompt_embeds [B, 77, D]
    replace the image embedding, :579-582) or on both (any other value: image token + text tokens concatenated, 78 keys, :583-587);
    per-frame mask `[B, F, 1, h, w]` duplicated for the two CFG halves (:590), conditioning latents either from the image
    (`_encode_vae_image`, zeros in the unconditional half, :598-601) or the caller's `condition_latent` [B, F, 4, h, w] used for both
    halves (:602-604); 9-channel UNets get cat([mask, x, cond]), 8-channel ones cat([x, cond]) (:657-660).
    The call the reference makes (app_svd.py:120-133) is condition_type="image" with `condition_latent` and a per-frame mask.  A
    multi-token context ("text" / both) is passed to the UNet as the reference does -- and fails there exactly as it does under
    the pinned diffusers 0.24, whose temporal transformer broadcasts the context with a literal 1 token (RuntimeError)."""

    @torch.no_grad()
    def __call__(self, image, prompt_embeds=None, negative_prompt_embeds=None, height: int = 576, width: int = 1024,
                 num_frames: Optional[int] = None, num_inference_steps: int = 25, min_guidance_scale: float = 1.0,
                 max_guidance_scale: float = 3.0, fps: int = 7, motion_bucket_id: int = 127, noise_aug_strength: float = 0.02,
                 decode_chunk_size: Optional[int] = None, num_videos_per_prompt: Optional[int] = 1,
                 generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
                 latents: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 callback_on_step_end: Optional[Callable[[int, int, Dict], None]] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"], return_dict: bool = True, mask=None,
                 condition_type="image", condition_latent=None, image_embeddings: Optional[torch.Tensor] = None):
        from . import _lib
        launches0 = _lib.launch_count()
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        num_frames = num_frames if num_frames is not None else self.unet.config.num_frames
        decode_chunk_size = decode_chunk_size if decode_chunk_size is not None else num_frames
        self.check_inputs(image, height, width)
        device, dtype = self.unet.device, self.unet.dtype
        cfg = max_guidance_scale > 1.0
        image_t = self.image_processor.preprocess(image, height=height, width=width).to(device)
        batch_size = image_t.shape[0]
        if batch_size * num_videos_per_prompt != 1:
            raise NotImplementedError("one video per call on the sm_90a path")

        def _text():
            if prompt_embeds is None or (cfg and negative_prompt_embeds is None):
                raise TypeError("condition_type != 'image' needs prompt_embeds (and negative_prompt_embeds under guidance)")
            pe = prompt_embeds.to(device=device, dtype=dtype)
            return torch.cat([negative_prompt_embeds.to(device=device, dtype=dtype), pe]) if cfg else pe

        def _img():
            if image_embeddings is None:
                return self._encode_image(image_t, device, num_videos_per_prompt, cfg)
            e = image_embeddings.to(device=device, dtype=dtype)
            return torch.cat([torch.zeros_like(e), e]) if cfg and e.shape[0] == batch_size else e

        if condition_type == "image":
            emb = _img()
        elif condition_type == "text":
            emb = _text()
        else:
            emb = torch.cat([_img(), _text()], dim=1)
        motion_mask = self.unet.config.in_channels == 9
        if cfg and mask is None:
            raise TypeError("expected Tensor as element 0 in argument 0, but got NoneType (torch.cat([mask] * 2), "
                            "models/pipeline.py:590)")
        fps = fps - 1
        noise = torch.randn(image_t.shape, generator=generator, device=generator.device if generator is not None else device,
                            dtype=image_t.dtype).to(device)
        image_t = image_t + noise_aug_strength * noise
        lat_h, lat_w = height // self.vae_scale_factor, width // self.vae_scale_factor
        if condition_latent is None:
            il = self.vae.encode(image_t.to(dtype)).latent_dist.mode().to(dtype).contiguous()          # [1, 4, h, w]
            cond = il.reshape(1, batch_size, 1, 4, lat_h, lat_w)
            zero_uncond = True
        else:
            cond = condition_latent.to(device=device, dtype=dtype).reshape(1, batch_size, num_frames, 4, lat_h, lat_w).contiguous()
            zero_uncond = False
        ids = torch.tensor([[fps, motion_bucket_id, noise_aug_strength]], dtype=dtype).repeat(batch_size, 1)
        ids = (torch.cat([ids, ids]) if cfg else ids).to(device)
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        timesteps = self.scheduler.timesteps
        sigmas = [float(s) for s in self.scheduler.sigmas]
        shape = (batch_size, num_frames, self.unet.config.in_channels // 2, lat_h, lat_w)
        if latents is None:
            latents = torch.randn(shape, generator=generator, device=generator.device if generator is not None else device,
                                  dtype=dtype).to(device)
        else:
            latents = latents.to(device=device, dtype=dtype)
        latents = (latents * float(self.scheduler.init_noise_sigma)).contiguous()
        gs = torch.linspace(min_guidance_scale, max_guidance_scale, num_frames).unsqueeze(0).to(device, latents.dtype)
        self._guidance_scale = _append_dims(gs.repeat(batch_size, 1), latents.ndim)
        gs_f32 = gs[0].float().contiguous()
        m16 = None
        if motion_mask:
            if mask is None:
                raise TypeError("a 9-channel UNet needs `mask` [B, F, 1, h, w] (models/pipeline.py:657)")
            if tuple(mask.shape) != (batch_size, num_frames, 1, lat_h, lat_w):
                raise RuntimeError(f"Sizes of tensors must match except in dimension 2: mask {tuple(mask.shape)} vs latents "
                                   f"{(batch_size, num_frames, 4, lat_h, lat_w)} (models/pipeline.py:657)")
            m16 = mask.to(device=device, dtype=dtype).reshape(batch_size, num_frames, lat_h, lat_w).contiguous()
        in_ch = self.unet.config.in_channels
        b_unet = (2 if cfg else 1) * batch_size
        self._num_timesteps = len(timesteps)
        for i, t in enumerate(timesteps):
            x16 = ops.svd_in_assemble_frames(latents, cond, m16, sigmas[i], cfg, zero_uncond)
            pred, _ = self.unet(None, t, emb, ids, _raw=True, _x16=x16, _shape=(b_unet, num_frames, in_ch, lat_h, lat_w))
            latents = ops.svd_cfg_euler_step(pred, cfg, gs_f32, latents, sigmas[i], sigmas[i + 1])
            if callback_on_step_end is not None:
                callback_kwargs = {k: locals()[k] for k in callback_on_step_end_tensor_inputs}
                callback_outputs = callback_on_step_end(self, i, t, callback_kwargs)
                latents = callback_outputs.pop("latents", latents)
        if output_type != "latent":
            frames = self.decode_latents(latents, num_frames, decode_chunk_size)
            frames = [self.image_processor.postprocess(frames[b].permute(1, 0, 2, 3), output_type)
                      for b in range(frames.shape[0])]
        else:
            frames = latents
        self.last_gpu_launches = _lib.launch_count() - launches0
        if not return_dict:
            return frames
        return StableVideoDiffusionPipelineOutput(frames=frames)
