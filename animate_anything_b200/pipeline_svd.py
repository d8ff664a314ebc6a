"""Mirror of diffusers 0.24 `StableVideoDiffusionPipeline` (loading, the stock image-to-video `__call__`) and of the
reference's `MaskStableVideoDiffusionPipeline.__call__` (models/pipeline.py:223-466; BASELINE config 4, driven by
train_svd.py:756-777) and `TextStableVideoDiffusionPipeline.__call__` (:468-731): same keyword arguments, defaults and
return values.  `output_type="pil"` frames are rounded to uint8 in the decoder's last kernel (`decode_chunk_frames_u8`).

What is mirrored on the sm_90a kernels (the hot path, reference line -> here):
  :359-362  `_encode_vae_image` (VAE encode of the noise-augmented image, `latent_dist.mode()`)  -> AutoencoderKLTemporalDecoder.encode
  :418-422  `cat([latents] * 2)`, `scale_model_input`, `cat([mask, x, image_latents], dim=2)`       -> ONE kernel, `aab_svd_in_assemble`
  :425-431  UNetSpatioTemporalConditionModel.forward                                              -> unet_spatio_temporal_condition.py
  :434-439  per-frame guidance (`linspace(min, max, F)`, :405-408) + EulerDiscreteScheduler.step  -> ONE kernel, `aab_svd_cfg_euler_step`
  :456      `decode_latents` in chunks of `decode_chunk_size` frames                                -> decode_chunk_video
  :347      `_encode_image` with a CLIP image tower (ours or a `transformers.CLIPVisionModelWithProjection`, mirrored once) on
            the caller's image, as diffusers 0.24 does: PIL -> resize with antialiasing to 224 + CLIP normalisation +
            patchify in ONE kernel (`aab_clip_image_prep`), then the ViT tower on the kernels (clip_vision.py); a tensor is
            taken as the CLIP pixel values
Any other `image_encoder` module (mapping the VAE-preprocessed image batch to `.image_embeds` or a tensor) is called as it is,
or pass `image_embeddings=`.
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


class StableVideoDiffusionPipeline:
    """Mirror of diffusers 0.24 `StableVideoDiffusionPipeline`, the object both SVD entry points build
    (`StableVideoDiffusionPipeline.from_pretrained(path, torch_dtype=torch.float16, variant="fp16")`, train_svd.py:87 and
    app_svd.py:37), and the base of the Mask / Text pipelines as in the reference (models/pipeline.py:223,468).  Everything
    their `__call__`s touch lives here, because the reference calls them unbound on a stock instance
    (`MaskStableVideoDiffusionPipeline.__call__(pipeline, ...)`, train_svd.py:766; `TextStableVideoDiffusionPipeline.__call__(
    self.pipeline, ...)`, app_svd.py:120)."""

    def __init__(self, vae, image_encoder, unet, scheduler, feature_extractor=None):
        self.vae, self.image_encoder, self.unet, self.scheduler = vae, image_encoder, unet, scheduler
        self.feature_extractor = feature_extractor
        self.vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
        from .image_processor import VaeImageProcessor
        self.image_processor = VaeImageProcessor(vae_scale_factor=self.vae_scale_factor)
        self.last_gpu_launches = 0

    @classmethod
    def from_pretrained(cls, path, torch_dtype=None, variant=None, unet=None, vae=None, image_encoder=None, scheduler=None,
                        feature_extractor=None):
        """Reads the diffusers SVD checkpoint layout: `unet/`, `vae/` (diffusers weight names), `image_encoder/`
        (transformers names, `model.safetensors`), `scheduler/scheduler_config.json` and
        `feature_extractor/preprocessor_config.json` (its `image_mean` / `image_std` are what the CLIP preprocessing
        reads).  `variant="fp16"` loads `*.fp16.safetensors` / `*.fp16.bin` weights.  A component passed as a keyword is
        used as it is instead of being loaded; a missing `image_encoder/` or `feature_extractor/` folder leaves None."""
        import json
        import os
        from .autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
        from .clip_vision import CLIPVisionModelWithProjection
        from .modeling import FrozenConfig
        from .schedulers import EulerDiscreteScheduler
        from .unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
        kw = dict(torch_dtype=torch_dtype, variant=variant)
        if unet is None:
            unet = UNetSpatioTemporalConditionModel.from_pretrained(path, subfolder="unet", **kw)
        if vae is None:
            vae = AutoencoderKLTemporalDecoder.from_pretrained(path, subfolder="vae", **kw)
        if image_encoder is None and os.path.isdir(os.path.join(path, "image_encoder")):
            image_encoder = CLIPVisionModelWithProjection.from_pretrained(path, subfolder="image_encoder", **kw)
        if scheduler is None:
            scheduler = EulerDiscreteScheduler.from_pretrained(path, subfolder="scheduler")
        fe_path = os.path.join(path, "feature_extractor", "preprocessor_config.json")
        if feature_extractor is None and os.path.exists(fe_path):
            with open(fe_path) as f:
                feature_extractor = FrozenConfig(json.load(f))
        return cls(vae=vae, image_encoder=image_encoder, unet=unet, scheduler=scheduler, feature_extractor=feature_extractor)

    def to(self, *args, device=None, dtype=None):
        """`pipeline.to("cuda")` / `.to(torch.float16)` / `.to(device=..., dtype=...)`: moves the UNet, VAE and image encoder."""
        for a in args:
            if isinstance(a, torch.dtype):
                dtype = a
            else:
                device = a
        for m in (self.vae, self.unet, self.image_encoder):
            if isinstance(m, torch.nn.Module):
                m.to(device=device, dtype=dtype)
        return self

    @property
    def device(self):
        return self.unet.device

    @property
    def dtype(self):
        return self.unet.dtype

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

    def _clip_image_encoder(self):
        """The image encoder as an sm_90a `clip_vision.CLIPVisionModelWithProjection`, or None when it is another module.
        A `transformers.CLIPVisionModelWithProjection` is mirrored once (same weights, dtype, device); the mirror is rebuilt
        if the caller swaps or moves the encoder."""
        from .clip_vision import CLIPVisionModelWithProjection
        enc = self.image_encoder
        if isinstance(enc, CLIPVisionModelWithProjection):
            return enc
        if type(enc).__name__ != "CLIPVisionModelWithProjection" or not type(enc).__module__.startswith("transformers"):
            return None
        p0 = next(enc.parameters())
        key = (id(enc), p0.data_ptr(), p0.dtype, p0.device)
        cached = self.__dict__.get("_ie_mirror")
        if cached is None or cached[0] != key:
            cached = (key, CLIPVisionModelWithProjection.from_hf(enc))
            self.__dict__["_ie_mirror"] = cached
        return cached[1]

    def _clip_image_embeds(self, enc, image, device):
        """diffusers 0.24 `_encode_image` up to `.image_embeds` on the caller's image: PIL images (or a list of them, or
        uint8 HWC arrays) go through `pil_to_numpy` -> [-1, 1] -> `_resize_with_antialiasing` -> [0, 1] -> the
        feature extractor's normalisation, all in `aab_clip_image_prep`; a tensor is the CLIP pixel values."""
        import numpy as np
        import PIL.Image
        from .clip_vision import OPENAI_CLIP_MEAN, OPENAI_CLIP_STD
        if isinstance(image, torch.Tensor):
            return enc(image.to(device)).image_embeds
        images = image if isinstance(image, list) else [image]
        arrs = []
        for im in images:
            if isinstance(im, PIL.Image.Image):
                if im.mode != "RGB":
                    raise ValueError(f"CLIP image encoding needs RGB images, got PIL mode {im.mode!r}")
                im = np.array(im)
            if not (isinstance(im, np.ndarray) and im.dtype == np.uint8 and im.ndim == 3 and im.shape[-1] == 3):
                raise NotImplementedError("CLIP image encoding takes PIL RGB images, uint8 [H, W, 3] arrays or CLIP pixel "
                                          "value tensors")
            arrs.append(im)
        u8 = torch.from_numpy(np.stack(arrs)).to(device)
        fe = self.feature_extractor
        mean = getattr(fe, "image_mean", None) or OPENAI_CLIP_MEAN
        std = getattr(fe, "image_std", None) or OPENAI_CLIP_STD
        return enc.encode_images(u8, mean, std).image_embeds

    def _encode_image(self, image, device, num_videos_per_prompt, do_classifier_free_guidance, raw_image=None):
        """CLIP image embedding [B, 1, D]; under CFG returns cat([zeros, embeddings]) (diffusers _encode_image).  A CLIP
        image tower encodes `raw_image`, the caller's image (models/pipeline.py:347 passes it before the VAE
        preprocessing); any other module gets `image`, the VAE-preprocessed batch."""
        dtype = self.unet.dtype
        enc = self._clip_image_encoder() if raw_image is not None else None
        if enc is not None:
            out = self._clip_image_embeds(enc, raw_image, device)
        else:
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
        chunks of `decode_chunk_size` frames of the flattened [B * F] axis (the temporal layers of the decoder see one chunk
        at a time; when the chunk size does not divide F, a chunk holds the last frames of one video and the first of the
        next, and they mix in those layers, as in diffusers)."""
        b = latents.shape[0]
        lat = latents.flatten(0, 1)
        outs = []
        inv = 1.0 / self.vae.config.scaling_factor
        for i in range(0, lat.shape[0], decode_chunk_size):
            z = lat[i: i + decode_chunk_size]
            # 1 / scaling_factor * latents: python float times 16-bit tensor -> one rounding (done by torch here: a scalar
            # scale of a [n, 4, h, w] latent, once per clip)
            z = (z * inv).contiguous()
            outs.append(self.vae.decode_chunk_video(z, z.shape[0]))           # [1, 3, n, H, W] fp32
        video = torch.cat(outs, dim=2)                                        # [1, 3, B*F, H, W]: chunks are consecutive frames
        return video.view(3, b, num_frames, *video.shape[-2:]).transpose(0, 1)    # [B, 3, F, H, W]

    def _output_frames(self, latents, num_frames, decode_chunk_size, output_type):
        """diffusers svd_tensor2vid(decode_latents(...), image_processor, output_type) -> one list / array / tensor of
        frames per video.  "pil" decodes each chunk straight to uint8 frames on the device (the decoder's last kernel
        rounds like `postprocess`), so one uint8 copy per chunk is all that reaches the host; the other types keep the
        fp32 video and `image_processor.postprocess`."""
        if output_type == "latent":
            return latents
        if output_type != "pil":
            frames = self.decode_latents(latents, num_frames, decode_chunk_size)
            return [self.image_processor.postprocess(frames[b].permute(1, 0, 2, 3), output_type)
                    for b in range(frames.shape[0])]                          # diffusers svd tensor2vid
        import PIL.Image
        lat = latents.flatten(0, 1)
        inv = 1.0 / self.vae.config.scaling_factor
        images = []
        for i in range(0, lat.shape[0], decode_chunk_size):
            z = (lat[i: i + decode_chunk_size] * inv).contiguous()          # as decode_latents
            u8 = self.vae.decode_chunk_frames_u8(z, z.shape[0]).cpu().numpy()   # [n, H, W, 3]
            images.extend(PIL.Image.fromarray(im) for im in u8)
        return [images[i: i + num_frames] for i in range(0, len(images), num_frames)]     # one list of frames per video

    def _check_text_batch_call(self, batch_size, num_frames, height, width, cfg, num_videos_per_prompt, generator, mask,
                               condition_latent, latents):
        """`TextStableVideoDiffusionPipeline.__call__` with B images: the errors the reference raises later (or a limit of the
        kernels), raised before the first launch.  On the base class because the reference calls the Text `__call__` unbound
        on a stock pipeline (app_svd.py:120)."""
        if num_videos_per_prompt != 1:
            # the reference repeats the embeddings and latents but not the mask / condition_latent, and its
            # torch.cat([mask, latent_model_input, condition_latent], dim=2) (:688) fails
            raise NotImplementedError("num_videos_per_prompt > 1 is not supported: pass the image several times instead")
        if isinstance(generator, list):
            raise TypeError("randn() received a list of generators; one torch.Generator seeds the whole image batch")
        lat = (height // self.vae_scale_factor, width // self.vae_scale_factor)
        motion_mask = self.unet.config.in_channels == 9
        if cfg and mask is None:
            raise TypeError("expected Tensor as element 0 in argument 0, but got NoneType (torch.cat([mask] * 2), "
                            "models/pipeline.py:609)")
        if motion_mask:
            if mask is None:
                raise TypeError("a 9-channel UNet needs `mask` [B, F, 1, h, w] (models/pipeline.py:688)")
            if tuple(mask.shape) != (batch_size, num_frames, 1) + lat:
                raise RuntimeError(f"Sizes of tensors must match except in dimension 2: mask {tuple(mask.shape)} vs latents "
                                   f"{(batch_size, num_frames, 4) + lat} (models/pipeline.py:688)")
        if condition_latent is not None and tuple(condition_latent.shape) != (batch_size, num_frames, 4) + lat:
            raise RuntimeError(f"Sizes of tensors must match except in dimension 2: condition_latent "
                               f"{tuple(condition_latent.shape)} vs latents {(batch_size, num_frames, 4) + lat} "
                               f"(models/pipeline.py:688-690)")
        want = (batch_size, num_frames, self.unet.config.in_channels // 2) + lat
        if latents is not None and tuple(latents.shape) != want:
            raise RuntimeError(f"Sizes of tensors must match except in dimension 2: latents {tuple(latents.shape)} vs "
                               f"{want} (models/pipeline.py:688-690)")
        unet_frames = (2 if cfg else 1) * batch_size * num_frames
        if unet_frames > ops.GN_MAX_SAMPLES:
            raise ValueError(f"the UNet batch holds {unet_frames} frames ((2 under guidance) x {batch_size} videos x "
                             f"{num_frames} frames); its GroupNorm kernel takes at most {ops.GN_MAX_SAMPLES}")

    @torch.no_grad()
    def __call__(self, image, height: int = 576, width: int = 1024, num_frames: Optional[int] = None,
                 num_inference_steps: int = 25, min_guidance_scale: float = 1.0, max_guidance_scale: float = 3.0,
                 fps: int = 7, motion_bucket_id: int = 127, noise_aug_strength: float = 0.02,
                 decode_chunk_size: Optional[int] = None, num_videos_per_prompt: Optional[int] = 1,
                 generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
                 latents: Optional[torch.Tensor] = None, output_type: Optional[str] = "pil",
                 callback_on_step_end: Optional[Callable[[int, int, Dict], None]] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"], return_dict: bool = True,
                 image_embeddings: Optional[torch.Tensor] = None):
        """diffusers 0.24 `StableVideoDiffusionPipeline.__call__` (image-to-video with an 8-channel UNet): the loop of the
        Mask call without the mask, i.e. `cat([latent_model_input, image_latents], dim=2)` with zeroed image latents in the
        unconditional half.  The input assembly, UNet, per-frame CFG + Euler step and temporal decode run on the sm_90a
        kernels.  One video per call.  Deviation: the stock call encodes the image with an fp32 VAE when
        `vae.config.force_upcast` (`needs_upcasting`); the sm_90a path is 16-bit, so the encode runs in the model dtype."""
        from . import _lib
        in_ch = self.unet.config.in_channels
        if in_ch != 8:
            raise ValueError(f"StableVideoDiffusionPipeline needs an 8-channel UNet (cat([latents, image_latents])), this one "
                             f"has in_channels={in_ch}; 9-channel motion-mask UNets go through "
                             "MaskStableVideoDiffusionPipeline / TextStableVideoDiffusionPipeline")
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
        if image_embeddings is None:
            image_embeddings = self._encode_image(image_t, device, num_videos_per_prompt, cfg, raw_image=image)
        else:
            image_embeddings = image_embeddings.to(device=device, dtype=dtype)
            if cfg and image_embeddings.shape[0] == batch_size:
                image_embeddings = torch.cat([torch.zeros_like(image_embeddings), image_embeddings])
        fps = fps - 1
        noise = torch.randn(image_t.shape, generator=generator, device=generator.device if generator is not None else device,
                            dtype=image_t.dtype).to(device)
        image_t = image_t + noise_aug_strength * noise
        lat_h, lat_w = height // self.vae_scale_factor, width // self.vae_scale_factor
        il = self.vae.encode(image_t.to(dtype)).latent_dist.mode().to(dtype).contiguous()              # [1, 4, h, w]
        cond = il.reshape(1, batch_size, 1, 4, lat_h, lat_w)
        ids = torch.tensor([[fps, motion_bucket_id, noise_aug_strength]], dtype=dtype).repeat(batch_size, 1)
        ids = (torch.cat([ids, ids]) if cfg else ids).to(device)
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        timesteps = self.scheduler.timesteps
        sigmas = [float(s) for s in self.scheduler.sigmas]
        shape = (batch_size, num_frames, in_ch // 2, lat_h, lat_w)
        if latents is None:
            latents = torch.randn(shape, generator=generator, device=generator.device if generator is not None else device,
                                  dtype=dtype).to(device)
        else:
            latents = latents.to(device=device, dtype=dtype)
        latents = (latents * float(self.scheduler.init_noise_sigma)).contiguous()
        gs = torch.linspace(min_guidance_scale, max_guidance_scale, num_frames).unsqueeze(0).to(device, latents.dtype)
        self._guidance_scale = _append_dims(gs.repeat(batch_size, 1), latents.ndim)
        gs_f32 = gs[0].float().contiguous()
        b_unet = (2 if cfg else 1) * batch_size
        self._num_timesteps = len(timesteps)
        for i, t in enumerate(timesteps):
            x16 = ops.svd_in_assemble_frames(latents, cond, None, sigmas[i], cfg, True)
            pred, _ = self.unet(None, t, image_embeddings, ids, _raw=True, _x16=x16,
                                _shape=(b_unet, num_frames, in_ch, lat_h, lat_w))
            latents = ops.svd_cfg_euler_step(pred, cfg, gs_f32, latents, sigmas[i], sigmas[i + 1])
            if callback_on_step_end is not None:
                callback_kwargs = {k: locals()[k] for k in callback_on_step_end_tensor_inputs}
                callback_outputs = callback_on_step_end(self, i, t, callback_kwargs)
                latents = callback_outputs.pop("latents", latents)
        frames = self._output_frames(latents, num_frames, decode_chunk_size, output_type)
        self.last_gpu_launches = _lib.launch_count() - launches0
        if not return_dict:
            return frames
        return StableVideoDiffusionPipelineOutput(frames=frames)


class MaskStableVideoDiffusionPipeline(StableVideoDiffusionPipeline):
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
        # 3. image embedding (once per clip) unless supplied
        image_t = self.image_processor.preprocess(image, height=height, width=width).to(device)
        batch_size = image_t.shape[0]
        if batch_size * num_videos_per_prompt != 1:
            raise NotImplementedError("the reference's mask handling ('1 h w -> 2 f 1 h w', :372) implies one video per call")
        if image_embeddings is None:
            image_embeddings = self._encode_image(image_t, device, num_videos_per_prompt, cfg, raw_image=image)
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
        frames = self._output_frames(latents, num_frames, decode_chunk_size, output_type)
        self.last_gpu_launches = _lib.launch_count() - launches0
        if not return_dict:
            return frames
        return StableVideoDiffusionPipelineOutput(frames=frames)


class TextStableVideoDiffusionPipeline(StableVideoDiffusionPipeline):
    """Mirror of the reference's `TextStableVideoDiffusionPipeline.__call__` (models/pipeline.py:468-731): the SVD loop
    conditioned on the CLIP image embedding (`condition_type="image"`), on text embeddings (`"text"`: prompt_embeds [B, 77, D]
    replace the image embedding, :579-582) or on both (any other value: image token + text tokens concatenated, 78 keys, :583-587);
    per-frame mask `[B, F, 1, h, w]` duplicated for the two CFG halves (:590), conditioning latents either from the image
    (`_encode_vae_image`, zeros in the unconditional half, :598-601) or the caller's `condition_latent` [B, F, 4, h, w] used for both
    halves (:602-604); 9-channel UNets get cat([mask, x, cond]), 8-channel ones cat([x, cond]) (:657-660).
    The call the reference makes (app_svd.py:120-133) is condition_type="image" with `condition_latent` and a per-frame mask.  A
    multi-token context ("text" / both) is passed to the UNet as the reference does -- and fails there exactly as it does under
    the pinned diffusers 0.24, whose temporal transformer broadcasts the context with a literal 1 token (RuntimeError).

    Several images make several videos in one call (`batch_size = len(image)`, :583-588): the CLIP tower and the VAE encode take
    the whole image batch, the UNet runs at batch 2B under guidance, and `decode_latents` decodes the flattened [B * F] frames in
    chunks of `decode_chunk_size`, so a chunk that does not divide F holds frames of two videos (see `decode_latents`)."""

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
        self._check_text_batch_call(batch_size, num_frames, height, width, cfg, num_videos_per_prompt, generator, mask,
                                    condition_latent, latents)

        def _text():
            if prompt_embeds is None or (cfg and negative_prompt_embeds is None):
                raise TypeError("condition_type != 'image' needs prompt_embeds (and negative_prompt_embeds under guidance)")
            pe = prompt_embeds.to(device=device, dtype=dtype)
            return torch.cat([negative_prompt_embeds.to(device=device, dtype=dtype), pe]) if cfg else pe

        def _img():
            if image_embeddings is None:
                return self._encode_image(image_t, device, num_videos_per_prompt, cfg, raw_image=image)
            e = image_embeddings.to(device=device, dtype=dtype)
            return torch.cat([torch.zeros_like(e), e]) if cfg and e.shape[0] == batch_size else e

        if condition_type == "image":
            emb = _img()
        elif condition_type == "text":
            emb = _text()
        else:
            emb = torch.cat([_img(), _text()], dim=1)
        motion_mask = self.unet.config.in_channels == 9
        fps = fps - 1
        noise = torch.randn(image_t.shape, generator=generator, device=generator.device if generator is not None else device,
                            dtype=image_t.dtype).to(device)
        image_t = image_t + noise_aug_strength * noise
        lat_h, lat_w = height // self.vae_scale_factor, width // self.vae_scale_factor
        if condition_latent is None:
            il = self.vae.encode(image_t.to(dtype)).latent_dist.mode().to(dtype).contiguous()          # [B, 4, h, w]
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
        frames = self._output_frames(latents, num_frames, decode_chunk_size, output_type)
        self.last_gpu_launches = _lib.launch_count() - launches0
        if not return_dict:
            return frames
        return StableVideoDiffusionPipelineOutput(frames=frames)
