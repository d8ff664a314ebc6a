"""Mirror of diffusers' `AutoencoderKL` (SD VAE) as the reference uses it:
  encode: utils/common.py:12-20 (`vae.encode(t).latent_dist.mode()`), train.py:747
  decode: models/pipeline.py:200 -> TextToVideoSDPipeline.decode_latents -> `vae.decode(latents).sample`
  surface: `.config.scaling_factor`, `.config.block_out_channels`, `.config.force_upcast`, `.enable_slicing()`,
           `.device`, `.dtype` (train.py:734-735,847; models/pipeline.py:359)
Same sub-module names as diffusers 0.24 (`encoder.down_blocks.i.resnets.j`, `mid_block.attentions.0.to_q`, ...), legacy
`query/key/value/proj_attn` checkpoint keys are converted on load.

All convolutions (3x3, stride-2, 1x1) run on the wgmma implicit-GEMM kernel over channels-last frames; GroupNorm+SiLU on
the fused norm kernels; the single-head (d=512) mid-block attention as two batched implicit GEMMs around a row softmax.
Frames are independent -> processed in chunks (`frame_chunk`) to bound the 128ch x 512^2 activations; `enable_slicing()`
is accepted and does not change results.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn as nn

from . import engine as E
from . import ops
from .layers import Attention, Downsample2D, ResnetBlock2D, Upsample2D
from .modeling import BaseOutput, ModelBase, capture_config


class DownEncoderBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_downsample, groups):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(in_channels=in_channels if i == 0 else out_channels,
                                                    out_channels=out_channels, temb_channels=None, eps=1e-6,
                                                    groups=groups) for i in range(num_layers)])
        self.downsamplers = (nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels,
                                                         padding=0, name="op")]) if add_downsample else None)


class UpDecoderBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_upsample, groups):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(in_channels=in_channels if i == 0 else out_channels,
                                                    out_channels=out_channels, temb_channels=None, eps=1e-6,
                                                    groups=groups) for i in range(num_layers)])
        self.upsamplers = (nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)])
                           if add_upsample else None)


class UNetMidBlock2D(nn.Module):
    def __init__(self, channels, groups):
        super().__init__()
        self.attentions = nn.ModuleList([Attention(channels, heads=1, dim_head=channels, bias=True,
                                                   norm_num_groups=groups, eps=1e-6, residual_connection=True)])
        self.resnets = nn.ModuleList([ResnetBlock2D(in_channels=channels, out_channels=channels, temb_channels=None,
                                                    eps=1e-6, groups=groups) for _ in range(2)])


class Encoder(nn.Module):
    def __init__(self, in_channels, latent_channels, block_out_channels, layers_per_block, groups):
        super().__init__()
        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], 3, padding=1)
        self.down_blocks = nn.ModuleList()
        out_c = block_out_channels[0]
        for i, c in enumerate(block_out_channels):
            in_c, out_c = out_c, c
            self.down_blocks.append(DownEncoderBlock2D(in_c, out_c, layers_per_block,
                                                       i != len(block_out_channels) - 1, groups))
        self.mid_block = UNetMidBlock2D(block_out_channels[-1], groups)
        self.conv_norm_out = nn.GroupNorm(groups, block_out_channels[-1], eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[-1], 2 * latent_channels, 3, padding=1)


class Decoder(nn.Module):
    def __init__(self, latent_channels, out_channels, block_out_channels, layers_per_block, groups):
        super().__init__()
        self.conv_in = nn.Conv2d(latent_channels, block_out_channels[-1], 3, padding=1)
        self.mid_block = UNetMidBlock2D(block_out_channels[-1], groups)
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(block_out_channels))
        out_c = rev[0]
        for i, c in enumerate(rev):
            prev, out_c = out_c, c
            self.up_blocks.append(UpDecoderBlock2D(prev, out_c, layers_per_block + 1, i != len(rev) - 1, groups))
        self.conv_norm_out = nn.GroupNorm(groups, block_out_channels[0], eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, 3, padding=1)


class DiagonalGaussianDistribution:
    def __init__(self, parameters: torch.Tensor):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)

    def mode(self):
        return self.mean

    def sample(self, generator=None):
        logvar = torch.clamp(self.logvar.float(), -30.0, 20.0)
        noise = torch.randn(self.mean.shape, generator=generator, device=self.mean.device, dtype=torch.float32)
        return (self.mean.float() + torch.exp(0.5 * logvar) * noise).to(self.mean.dtype)


class AutoencoderKLOutput(BaseOutput):
    pass


class DecoderOutput(BaseOutput):
    pass


class AutoencoderKL(ModelBase):
    def __init__(self, in_channels: int = 3, out_channels: int = 3,
                 down_block_types: Tuple[str] = ("DownEncoderBlock2D",) * 4,
                 up_block_types: Tuple[str] = ("UpDecoderBlock2D",) * 4,
                 block_out_channels: Tuple[int] = (128, 256, 512, 512), layers_per_block: int = 2,
                 act_fn: str = "silu", latent_channels: int = 4, norm_num_groups: int = 32, sample_size: int = 512,
                 scaling_factor: float = 0.18215, force_upcast: bool = True):
        super().__init__()
        capture_config(self, AutoencoderKL.__init__, (), dict(
            in_channels=in_channels, out_channels=out_channels, down_block_types=down_block_types,
            up_block_types=up_block_types, block_out_channels=block_out_channels, layers_per_block=layers_per_block,
            act_fn=act_fn, latent_channels=latent_channels, norm_num_groups=norm_num_groups, sample_size=sample_size,
            scaling_factor=scaling_factor, force_upcast=force_upcast))
        if latent_channels != 4 or in_channels != 3 or out_channels != 3:
            raise ValueError("specialised for the SD VAE: 3 image channels, 4 latent channels")
        if any(c % 64 for c in block_out_channels):
            raise ValueError("block_out_channels must be multiples of 64 (implicit-GEMM K tiles)")
        self.encoder = Encoder(in_channels, latent_channels, block_out_channels, layers_per_block, norm_num_groups)
        self.decoder = Decoder(latent_channels, out_channels, block_out_channels, layers_per_block, norm_num_groups)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
        self.use_slicing = False
        self.frame_chunk = 8
        self.__dict__["_aab_prepared"] = None

    def enable_slicing(self):
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    def _convert_legacy_keys(self, sd):
        out = {}
        ren = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}
        for k, v in sd.items():
            parts = k.split(".")
            if "attentions" in parts and len(parts) >= 2 and parts[-2] in ren:
                parts[-2] = ren[parts[-2]]
                k = ".".join(parts)
                if v.dim() == 4:
                    v = v[:, :, 0, 0]
            out[k] = v
        return out

    # ------------------------------------------------------------------ weights
    def _prepared(self) -> E.Prepared:
        prep = self.__dict__.get("_aab_prepared")
        p0 = self.quant_conv.weight
        if prep is not None and prep.dtype == p0.dtype and prep.device == p0.device:
            return prep
        if p0.dtype not in (torch.float16, torch.bfloat16) or not p0.is_cuda:
            raise TypeError("AutoencoderKL must be fp16/bf16 on a CUDA device for the sm_90a path (no fallback)")
        prep = self._build_prepared(p0.dtype, p0.device)
        self.__dict__["_aab_prepared"] = prep
        return prep

    def _build_prepared(self, dt, device) -> E.Prepared:
        prep = E.Prepared(dt, device)
        with torch.no_grad():
            E.prepare_module(prep, self)
            own = {
                "enc_in": E.prep_conv3x3(self.encoder.conv_in, dt, pad_cin_to=8),
                "enc_norm": E.prep_norm(self.encoder.conv_norm_out),
                "enc_out": E.prep_conv3x3(self.encoder.conv_out, dt),
                "dec_in": E.prep_conv3x3(self.decoder.conv_in, dt, pad_cin_to=8),
                "dec_norm": E.prep_norm(self.decoder.conv_norm_out),
                "dec_out": E.prep_conv3x3(self.decoder.conv_out, dt),
                "quant": (self.quant_conv.weight.detach().float().reshape(8, 8).contiguous(),
                          self.quant_conv.bias.detach().float().contiguous()),
                "post_quant": (self.post_quant_conv.weight.detach().float().reshape(4, 4).contiguous(),
                               self.post_quant_conv.bias.detach().float().contiguous()),
            }
            prep.put(self, own)
        return prep

    # ------------------------------------------------------------------ engine pieces
    def _mid_attention(self, ctx, attn: Attention, x: torch.Tensor, g: E.Geo):
        """diffusers Attention (deprecated attn-block form): GroupNorm -> q,k,v (bias) -> softmax(QK^T/sqrt(C))V ->
        to_out -> + residual.  One head of dim C: S and O are batched implicit GEMMs, softmax in fp32 (upcast_softmax)."""
        p = ctx.prep.get(attn)
        c = attn.inner_dim
        hn = ops.groupnorm(x, g.n, g.hw, p["gn"][0], p["gn"][1], 1e-6, False, 32)
        qkv = ops.linear(hn, p["qkv"], p["qkv_b"])                       # [n*l, 3c]
        o = ops.single_head_attention(qkv, g.n, g.hw, c)
        return ops.linear(o, p["o"][0], p["o"][1], residual=x, out_scale=1.0 / attn.rescale_output_factor, stats=True)

    def _mid(self, ctx, mid: UNetMidBlock2D, x, g):
        x = E.resnet_forward(ctx, mid.resnets[0], x, g)
        x = self._mid_attention(ctx, mid.attentions[0], x, g)
        return E.resnet_forward(ctx, mid.resnets[1], x, g)

    def _encode_chunk(self, prep, x: torch.Tensor, bf=None, scale: float = 1.0) -> torch.Tensor:
        """x [n, 3, H, W] -> moments [n, 8, h, w]; with bf=(b, f) (n = b*f) -> scaled moments [b, 8, f, h, w]."""
        own = prep.get(self)
        n, _, hh, ww = x.shape
        if hh % 8 or ww % 8:
            raise ValueError("image height/width must be multiples of 8")
        g = E.Geo(n, 1, hh, ww)
        ctx = E.Ctx(prep, g)
        h = ops.conv3x3(ops.image_to_nhwc8(x), own["enc_in"][0], own["enc_in"][1], stats=True)
        for blk in self.encoder.down_blocks:
            for r in blk.resnets:
                h = E.resnet_forward(ctx, r, h, g)
            if blk.downsamplers is not None:
                h = E.downsample_forward(ctx, blk.downsamplers[0], h, g, pad_mode="br")
                g = g.down()
        h = self._mid(ctx, self.encoder.mid_block, h, g)
        c_last = self.encoder.conv_out.in_channels
        h = ops.groupnorm(h, g.n, g.hw, own["enc_norm"][0], own["enc_norm"][1], 1e-6, True, 32)
        mom = ops.conv3x3(h.view(g.n, g.h, g.w, c_last), own["enc_out"][0], own["enc_out"][1])   # [rows, 8]
        if bf is not None:
            return ops.vae_enc_finalize(mom, own["quant"][0], own["quant"][1], scale, bf[0], bf[1], g.h, g.w)
        return ops.vae_enc_finalize(mom, own["quant"][0], own["quant"][1], 1.0, n, 1, g.h, g.w)[:, :, 0]

    def _decode_chunk(self, prep, lat5: torch.Tensor, inv_scale: float, as_uint8: bool = False) -> torch.Tensor:
        """lat5 [b, 4, f, h, w] (already divided by scaling unless inv_scale != 1) -> fp32 [b, 3, f, 8h, 8w]
        (or uint8 frames [f, 8h, b*8w, 3] when `as_uint8`)."""
        own = prep.get(self)
        b, _, f, hh, ww = lat5.shape
        g = E.Geo(b * f, 1, hh, ww)
        ctx = E.Ctx(prep, g)
        z = ops.vae_dec_in(lat5, inv_scale, own["post_quant"][0], own["post_quant"][1])
        h = ops.conv3x3(z, own["dec_in"][0], own["dec_in"][1], stats=True)
        h = self._mid(ctx, self.decoder.mid_block, h, g)
        for blk in self.decoder.up_blocks:
            for r in blk.resnets:
                h = E.resnet_forward(ctx, r, h, g)
            if blk.upsamplers is not None:
                h = E.upsample_forward(ctx, blk.upsamplers[0], h, g)
                g = g.up()
        c0 = self.decoder.conv_out.in_channels
        h = ops.groupnorm(h, g.n, g.hw, own["dec_norm"][0], own["dec_norm"][1], 1e-6, True, 32)
        y = ops.conv3x3(h.view(g.n, g.h, g.w, c0), own["dec_out"][0], own["dec_out"][1], out_f32=True)   # [rows, 3]
        if as_uint8 == "both":         # MaskedLatentToVideoPipeline needs the fp32 video (alpha decoder input) AND the frames
            return (ops.vae_dec_finalize(y, b, f, g.h, g.w, prep.dtype == torch.bfloat16),
                    ops.vae_dec_finalize_u8(y, b, f, g.h, g.w, prep.dtype == torch.bfloat16))
        if as_uint8:
            return ops.vae_dec_finalize_u8(y, b, f, g.h, g.w, prep.dtype == torch.bfloat16)
        return ops.vae_dec_finalize(y, b, f, g.h, g.w, prep.dtype == torch.bfloat16)

    # ------------------------------------------------------------------ public API (diffusers surface)
    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        prep = self._prepared()
        x = x.to(prep.dtype)
        chunks = [self._encode_chunk(prep, x[i: i + self.frame_chunk]) for i in range(0, x.shape[0], self.frame_chunk)]
        moments = chunks[0] if len(chunks) == 1 else torch.cat(chunks, dim=0)
        posterior = DiagonalGaussianDistribution(moments)
        if not return_dict:
            return (posterior,)
        return AutoencoderKLOutput(latent_dist=posterior)

    @torch.no_grad()
    def encode_video_latents(self, frames: torch.Tensor, scale: float = 0.18215) -> torch.Tensor:
        """Fused `tensor_to_vae_latent` (utils/common.py:12-20): frames [b, f, 3, H, W] -> `latent_dist.mode() * scale`
        laid out [b, 4, f, h, w]; the two rearranges and the scaling happen inside the quant_conv kernel (with the
        reference's two 16-bit roundings)."""
        prep = self._prepared()
        b, f = frames.shape[:2]
        x = frames.to(prep.dtype).reshape(b * f, *frames.shape[2:])
        if f <= self.frame_chunk:
            return self._encode_chunk(prep, x, bf=(b, f), scale=scale)[:, :4].contiguous()
        outs = [self._encode_chunk(prep, frames[:, i: i + self.frame_chunk].to(prep.dtype).reshape(-1, *frames.shape[2:]),
                                   bf=(b, min(self.frame_chunk, f - i)), scale=scale)[:, :4]
                for i in range(0, f, self.frame_chunk)]
        return torch.cat(outs, dim=2).contiguous()

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        """z [N, 4, h, w] -> image [N, 3, 8h, 8w] in the model dtype (diffusers semantics)."""
        video = self.decode_video(z.unsqueeze(0).permute(0, 2, 1, 3, 4), inv_scale=1.0)      # [1, 3, N, H, W] fp32
        img = video[0].permute(1, 0, 2, 3).to(z.dtype if z.dtype in (torch.float16, torch.bfloat16) else self.dtype)
        if not return_dict:
            return (img,)
        return DecoderOutput(sample=img)

    @torch.no_grad()
    def decode_video(self, latents: torch.Tensor, inv_scale: Optional[float] = None, frame_slice=None) -> torch.Tensor:
        """Fused decode_latents: latents [b, 4, f, h, w] -> fp32 video [b, 3, f, 8h, 8w]; frames in chunks."""
        prep = self._prepared()
        if inv_scale is None:
            inv_scale = 1.0 / self.config.scaling_factor
        latents = latents.to(prep.dtype).contiguous()
        b, _, f, h, w = latents.shape
        outs = []
        for i in range(0, f, self.frame_chunk):
            outs.append(self._decode_chunk(prep, latents[:, :, i: i + self.frame_chunk].contiguous(), inv_scale))
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=2)

    @torch.no_grad()
    def decode_frames_uint8(self, latents: torch.Tensor, inv_scale: Optional[float] = None) -> torch.Tensor:
        """decode_latents + tensor2vid fused: latents [b, 4, f, h, w] -> uint8 frames [f, 8h, b*8w, 3] on the device."""
        prep = self._prepared()
        if inv_scale is None:
            inv_scale = 1.0 / self.config.scaling_factor
        latents = latents.to(prep.dtype).contiguous()
        f = latents.shape[2]
        outs = [self._decode_chunk(prep, latents[:, :, i: i + self.frame_chunk].contiguous(), inv_scale, as_uint8=True)
                for i in range(0, f, self.frame_chunk)]
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)

    @torch.no_grad()
    def decode_video_and_frames_uint8(self, latents: torch.Tensor, inv_scale: Optional[float] = None):
        """One decoder pass, both tails: (fp32 video [b, 3, f, H, W], uint8 tensor2vid frames [f, H, b*W, 3]) — what
        models/pipeline_stage2.py:299 (`decode_latents`) and :330 (`tensor2vid`) produce from the same latents."""
        prep = self._prepared()
        if inv_scale is None:
            inv_scale = 1.0 / self.config.scaling_factor
        latents = latents.to(prep.dtype).contiguous()
        f = latents.shape[2]
        outs = [self._decode_chunk(prep, latents[:, :, i: i + self.frame_chunk].contiguous(), inv_scale, as_uint8="both")
                for i in range(0, f, self.frame_chunk)]
        if len(outs) == 1:
            return outs[0]
        return torch.cat([o[0] for o in outs], dim=2), torch.cat([o[1] for o in outs], dim=0)
