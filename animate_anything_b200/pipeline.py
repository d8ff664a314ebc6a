"""Mirror of the reference's `models/pipeline.py` `LatentToVideoPipeline.__call__` (:14-214): same keyword
arguments, same return values (`return_dict=False` -> `(video, latents)`), same semantics — classifier-free guidance with
cat([negative, positive]) embeddings (:136,:161,:165), caller-supplied truncated `timesteps` (:149-152), motion value
(:167-168), CFG combine (:180-181), scheduler step on `(b f) c h w` (:184-192), VAE decode (:200), tensor2vid (:205).

What changes is *how* a step executes:
  * the CFG-duplicated latent batch is a stride-0 view, never `torch.cat([latents] * 2)`;
  * cross-attention K/V of the (constant) prompt embeddings are projected once per call, not once per step;
  * UNet output (fp32, channels-last) -> CFG combine -> scheduler step -> next latents is ONE kernel;
  * with `use_cuda_graph=True` the whole step (≈1.2k kernel launches) is captured once and replayed per step; timestep
    and coefficient row are read from device memory indexed by a device-side step counter.
Multi-GPU (`parallel.py`): batch elements (CFG halves / prompts) and VAE frames are sharded, decoded frames gathered with
one NCCL all-gather.
"""
from __future__ import annotations

from typing import List, Optional, Union

import numpy as np
import torch

from . import ops
from .modeling import BaseOutput


class TextToVideoSDPipelineOutput(BaseOutput):
    pass


def tensor2vid(video: torch.Tensor, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)) -> List[np.ndarray]:
    """diffusers tensor2vid (models/pipeline.py:205): [-1,1] float video [b,c,f,h,w] -> list of f uint8 frames [h, b*w, c]."""
    m = torch.tensor(mean, device=video.device).reshape(1, -1, 1, 1, 1)
    s = torch.tensor(std, device=video.device).reshape(1, -1, 1, 1, 1)
    video = video.mul(s).add_(m).clamp_(0, 1)
    i, c, f, h, w = video.shape
    images = video.permute(2, 3, 0, 4, 1).reshape(f, h, i * w, c)
    return [(img.cpu().numpy() * 255).astype("uint8") for img in images.unbind(dim=0)]


class LatentToVideoPipeline:
    def __init__(self, vae, text_encoder, tokenizer, unet, scheduler):
        self.vae, self.text_encoder, self.tokenizer, self.unet, self.scheduler = vae, text_encoder, tokenizer, unet, scheduler
        self.vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1) if vae is not None else 8
        self.use_cuda_graph = True     # replay the captured step (bit-identical to eager; INTEGRATION.md section 4)
        self.share_cfg_prefix = True   # evaluate the text-independent prefix of the UNet once per CFG pair
        self.cfg_group = None          # torch.distributed group of size 2: CFG halves split over two GPUs (parallel.py)
        self.last_gpu_launches = 0

    @classmethod
    def from_pretrained(cls, path, text_encoder=None, vae=None, unet=None, scheduler=None, tokenizer=None, **kw):
        """models/pipeline.py / train.py:799: components given by the caller are used as-is; missing ones are loaded."""
        import json
        import os
        from .autoencoder_kl import AutoencoderKL
        from .unet_3d_condition_mask import UNet3DConditionModel
        from . import schedulers as S
        if unet is None:
            unet = UNet3DConditionModel.from_pretrained(path, subfolder="unet")
        if vae is None:
            vae = AutoencoderKL.from_pretrained(path, subfolder="vae")
        if scheduler is None:
            with open(os.path.join(path, "scheduler", "scheduler_config.json")) as f:
                cfg = json.load(f)
            klass = getattr(S, cfg.get("_class_name", "DDIMScheduler"), S.DDIMScheduler)
            scheduler = klass.from_config({k: v for k, v in cfg.items() if not k.startswith("_")})
        if tokenizer is None and os.path.isdir(os.path.join(path, "tokenizer")):
            from transformers import CLIPTokenizer
            tokenizer = CLIPTokenizer.from_pretrained(path, subfolder="tokenizer")
        if text_encoder is None and os.path.isdir(os.path.join(path, "text_encoder")):
            from .clip_text import CLIPTextModel
            text_encoder = CLIPTextModel.from_pretrained(path, subfolder="text_encoder")
        return cls(vae=vae, text_encoder=text_encoder, tokenizer=tokenizer, unet=unet, scheduler=scheduler)

    def to(self, device=None, dtype=None):
        for m in (self.vae, self.unet, self.text_encoder):
            if m is not None:
                m.to(device=device, dtype=dtype)
        return self

    # ------------------------------------------------------------------ helpers mirrored from TextToVideoSDPipeline
    def check_inputs(self, prompt, height, width, callback_steps, negative_prompt=None, prompt_embeds=None,
                     negative_prompt_embeds=None):
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        if (callback_steps is None) or (not isinstance(callback_steps, int) or callback_steps <= 0):
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps}.")
        if prompt is not None and prompt_embeds is not None:
            raise ValueError("Cannot forward both `prompt` and `prompt_embeds`.")
        if prompt is None and prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both undefined.")
        if prompt is not None and not isinstance(prompt, (str, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if negative_prompt is not None and negative_prompt_embeds is not None:
            raise ValueError("Cannot forward both `negative_prompt` and `negative_prompt_embeds`.")
        if prompt_embeds is not None and negative_prompt_embeds is not None and \
                prompt_embeds.shape != negative_prompt_embeds.shape:
            raise ValueError("`prompt_embeds` and `negative_prompt_embeds` must have the same shape")

    def _b200_text_encoder(self):
        """The text encoder as an sm_90a `clip_text.CLIPTextModel`.  A `transformers.CLIPTextModel` handed in by the
        caller (train.py:88,799 does exactly that) is mirrored once (same weights, dtype, device) so that prompt strings
        never run a library GEMM / SDPA; the mirror is rebuilt if the caller swaps or moves the encoder."""
        from .clip_text import CLIPTextModel
        te = self.text_encoder
        if te is None or isinstance(te, CLIPTextModel):
            return te
        if not (hasattr(te, "text_model") and hasattr(te, "config") and hasattr(te, "parameters")):
            return te                    # not a CLIP text model (a caller-supplied embedding callable): used as it is
        p0 = next(te.parameters())
        key = (id(te), p0.data_ptr(), p0.dtype, p0.device)
        cached = self.__dict__.get("_te_mirror")
        if cached is None or cached[0] != key:
            cached = (key, CLIPTextModel.from_hf(te))
            self.__dict__["_te_mirror"] = cached
        return cached[1]

    def _encode_prompt(self, prompt, device, num_images_per_prompt, do_cfg, negative_prompt=None, prompt_embeds=None,
                       negative_prompt_embeds=None, lora_scale=None):
        """diffusers TextToVideoSDPipeline._encode_prompt: CLIP text states; under CFG returns cat([negative, positive]).
        The CLIP forward runs on the sm_90a kernels (clip_text.py)."""
        def embed(texts):
            if self.text_encoder is None or self.tokenizer is None:
                raise ValueError("prompt strings need a text_encoder/tokenizer; pass prompt_embeds instead")
            tok = self.tokenizer(texts, padding="max_length", max_length=self.tokenizer.model_max_length,
                                 truncation=True, return_tensors="pt")
            return self._b200_text_encoder()(tok.input_ids.to(device))[0]
        if prompt_embeds is None:
            prompt_embeds = embed([prompt] if isinstance(prompt, str) else prompt)
        dtype = self.unet.dtype
        prompt_embeds = prompt_embeds.to(dtype=dtype, device=device)
        if do_cfg:
            if negative_prompt_embeds is None:
                n = prompt_embeds.shape[0]
                neg = [""] * n if negative_prompt is None else ([negative_prompt] * n if isinstance(negative_prompt, str)
                                                                else negative_prompt)
                negative_prompt_embeds = embed(neg)
            negative_prompt_embeds = negative_prompt_embeds.to(dtype=dtype, device=device)
            prompt_embeds = torch.cat([negative_prompt_embeds, prompt_embeds])
        return prompt_embeds

    def decode_latents(self, latents):
        """TextToVideoSDPipeline.decode_latents: [b,4,f,h,w] -> float32 video [b,3,f,H,W] in [-1, 1]."""
        return self.vae.decode_video(latents)

    # ------------------------------------------------------------------ the loop
    def _one_step(self, latents_in, latents_out, t_dev, ehs, cond2, mask, motion_dev, cfg, guidance, coef_row, step_idx,
                  x0_hist, kv_cache):
        n = latents_in.shape[0]
        if cfg and self.cfg_group is not None:
            # CFG halves on two GPUs (SURVEY 8e): rank 0 of the pair runs the unconditional half, rank 1 the text half;
            # the fp32 noise predictions (4 B x 4 x T x h x w per half) are all-gathered, then both ranks apply the
            # same fused CFG + scheduler step, so the latents stay bit-identical on the two GPUs.
            import torch.distributed as dist
            r = dist.get_rank(self.cfg_group)
            eps_half, g = self.unet(latents_in, t_dev, ehs[r * n:(r + 1) * n], condition_latent=cond2[r * n:(r + 1) * n],
                                    mask=mask, motion=motion_dev, _raw_eps=True, _kv_cache=kv_cache)
            eps = torch.empty((2,) + tuple(eps_half.shape), dtype=eps_half.dtype, device=eps_half.device)
            dist.all_gather_into_tensor(eps, eps_half.unsqueeze(0), group=self.cfg_group)
            eps = eps.view(2 * eps_half.shape[0], eps_half.shape[1])
        elif cfg and self.share_cfg_prefix:
            # both guidance halves share latents / condition / timestep: the UNet evaluates the layers before the first
            # text cross-attention once (cond2[:n] is the single copy of the condition latent)
            eps, g = self.unet(latents_in, t_dev, ehs, condition_latent=cond2[:n], mask=mask, motion=motion_dev,
                               _raw_eps=True, _kv_cache=kv_cache, _cfg_shared_prefix=True)
        else:
            if not cfg:
                sample = latents_in
            elif n == 1:
                sample = latents_in.expand(2, *latents_in.shape[1:])          # stride-0 duplicate, no copy
            else:
                sample = torch.cat([latents_in, latents_in])                  # multi-prompt: [uncond..., text...]
            eps, g = self.unet(sample, t_dev, ehs, condition_latent=cond2, mask=mask, motion=motion_dev, _raw_eps=True,
                               _kv_cache=kv_cache)
        ops.cfg_scheduler_step(eps, eps.stride(0), cfg, guidance, latents_in, latents_out, x0_hist, coef_row, step_idx)

    @torch.no_grad()
    def __call__(self, prompt=None, height=None, width=None, num_frames: int = 16, num_inference_steps: int = 50,
                 guidance_scale=9.0, negative_prompt=None, eta: float = 0.0, generator=None, latents=None,
                 prompt_embeds=None, negative_prompt_embeds=None, output_type="np", return_dict: bool = True,
                 callback=None, callback_steps: int = 1, cross_attention_kwargs=None, condition_latent=None, mask=None,
                 timesteps=None, motion=None):
        from . import _lib
        launches0 = _lib.launch_count()
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        self.check_inputs(prompt, height, width, callback_steps, negative_prompt, prompt_embeds, negative_prompt_embeds)
        if latents is None or condition_latent is None:
            raise ValueError("LatentToVideoPipeline needs `latents` and `condition_latent` (models/pipeline.py:126,161)")
        device = latents.device
        dtype = self.unet.dtype
        cfg = guidance_scale > 1.0
        ehs = self._encode_prompt(prompt, device, 1, cfg, negative_prompt, prompt_embeds=prompt_embeds,
                                  negative_prompt_embeds=negative_prompt_embeds)
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        if timesteps is None:
            timesteps = self.scheduler.timesteps
        ts_list = [int(t) for t in (timesteps.tolist() if torch.is_tensor(timesteps) else timesteps)]
        coef_np, needs_hist = self.scheduler.step_coefficients(ts_list, eta=eta)
        coef = torch.from_numpy(coef_np).to(device)
        t_table = torch.tensor(ts_list, dtype=torch.float32, device=device)

        latents = latents.to(dtype).contiguous()
        cond = condition_latent.to(dtype)
        cond2 = torch.cat([cond, cond]) if cfg else cond
        if mask is not None:
            mask = mask.to(dtype)
        motion_dev = None if motion is None else torch.tensor(motion, dtype=torch.float32, device=device).reshape(-1)
        x0_hist = torch.zeros(latents.shape, dtype=torch.float32, device=device) if needs_hist else None
        kv_cache = {}

        if self.use_cuda_graph:
            latents = self._run_graphed([latents], t_table, ehs, cond2, mask, motion_dev, cfg, float(guidance_scale),
                                        coef, x0_hist, kv_cache, callback, callback_steps, ts_list)
        else:
            # ping-pong between two scratch buffers; the caller's `latents` tensor is only ever read
            buf = [torch.empty_like(latents), torch.empty_like(latents)]
            src = latents
            for i, t in enumerate(ts_list):
                dst = buf[i & 1]
                self._one_step(src, dst, t_table[i: i + 1], ehs, cond2, mask, motion_dev, cfg,
                               float(guidance_scale), coef[i], None, x0_hist, kv_cache)
                src = dst
                if callback is not None and i % callback_steps == 0:
                    callback(i, t, dst)
            latents = src

        if output_type == "pt":
            video = self.decode_latents(latents)
        elif output_type == "latent":
            video = latents
        elif output_type == "u8":
            # extension used by parallel.py / bench.py: the tensor2vid frames as ONE device tensor [f, H, b*W, 3] uint8
            # (what "np" returns, before the D2H copy), ready for the NCCL all-gather
            video = self.vae.decode_frames_uint8(latents)
        else:
            # decode_latents + tensor2vid fused on the device (uint8 frames, 4x less D2H traffic than the fp32 video)
            frames = self.vae.decode_frames_uint8(latents).cpu().numpy()
            video = [frames[i] for i in range(frames.shape[0])]
        self.last_gpu_launches = _lib.launch_count() - launches0
        if not return_dict:
            return (video, latents)
        return TextToVideoSDPipelineOutput(frames=video)

    # ------------------------------------------------------------------ CUDA-graph replay of the step
    def _run_graphed(self, buf, t_table, ehs, cond2, mask, motion_dev, cfg, guidance, coef, x0_hist, kv_cache, callback,
                     callback_steps, ts_list):
        """Capture two graphs (even step: lat0->lat1, odd step: lat1->lat0) once per shape and replay them.  Timestep and
        coefficient row live in small device buffers refreshed by a memcpy before each replay; prompt / condition / mask
        inputs are copied into the captured static buffers, so a new call with the same shapes re-uses the graphs.
        (Text K/V projections are recomputed inside the captured step: 16 tiny GEMMs.)"""
        dev = buf[0].device
        # the captured kernels hold raw pointers into the UNet's converted weights (`Prepared`): its generation number is
        # part of the key, so `load_state_dict()` / `.to()` / `invalidate_prepared()` (which drop that cache) force a
        # re-capture instead of replaying graphs over freed memory.  In-place edits of parameters (e.g. a LoRA merge)
        # do not touch the cache: call `unet.invalidate_prepared()` after them.
        key = (tuple(buf[0].shape), buf[0].dtype, tuple(ehs.shape), cfg, guidance, mask is not None,
               motion_dev is not None, x0_hist is not None, bool(self.share_cfg_prefix), id(self.cfg_group),
               self.unet._prepared().gen)
        st = self.__dict__.get("_gstate")
        if st is None or st["key"] != key:
            st = {"key": key}
            st["lat"] = [torch.empty_like(buf[0]), torch.empty_like(buf[0])]
            st["t_cur"] = torch.zeros(1, dtype=torch.float32, device=dev)
            st["coef_cur"] = torch.zeros(6, dtype=torch.float32, device=dev)
            st["ehs"] = ehs.clone()
            st["cond2"] = cond2.clone()
            st["mask"] = None if mask is None else mask.clone()
            st["motion"] = None if motion_dev is None else motion_dev.clone()
            st["hist"] = None if x0_hist is None else torch.zeros_like(x0_hist)

            def step(par):
                self._one_step(st["lat"][par], st["lat"][1 - par], st["t_cur"], st["ehs"], st["cond2"], st["mask"],
                               st["motion"], cfg, guidance, st["coef_cur"], None, st["hist"], None)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):          # warm-up: lazy weight prep, smem attributes, allocator
                st["lat"][0].copy_(buf[0])
                step(0)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            st["graphs"] = []
            from . import _lib
            for par in (0, 1):
                gph = torch.cuda.CUDAGraph()
                c0 = _lib.launch_count()
                with torch.cuda.graph(gph):
                    step(par)
                self.graph_kernels_per_step = _lib.launch_count() - c0     # kernels re-launched by every replay
                st["graphs"].append(gph)
            self.__dict__["_gstate"] = st
        else:
            st["ehs"].copy_(ehs)
            st["cond2"].copy_(cond2)
            if mask is not None:
                st["mask"].copy_(mask)
            if motion_dev is not None:
                st["motion"].copy_(motion_dev)
        if st["hist"] is not None:
            st["hist"].zero_()
        st["lat"][0].copy_(buf[0])
        for i, t in enumerate(ts_list):
            st["t_cur"].copy_(t_table[i: i + 1], non_blocking=True)
            st["coef_cur"].copy_(coef[i], non_blocking=True)
            st["graphs"][i & 1].replay()
            if callback is not None and i % callback_steps == 0:
                callback(i, t, st["lat"][(i + 1) & 1])
        return st["lat"][len(ts_list) & 1].clone()
