"""Mirror of diffusers' `AutoencoderKLTemporalDecoder` (the SVD VAE) as the reference uses it:
`MaskStableVideoDiffusionPipeline.__call__` encodes the conditioning image (`_encode_vae_image`, models/pipeline.py:359-362)
and decodes the final latents in chunks of `decode_chunk_size` frames (`decode_latents`, :456).

Encoder = the SD VAE encoder (shared code with autoencoder_kl.py).  Decoder = `TemporalDecoder`: every res block is a
SpatioTemporalResBlock without time embedding (merge "learned", switched: alpha = 1 - sigmoid(mix_factor)), the mid block
carries the single-head d=512 attention, and a final Conv3d(3, 3, (3,1,1)) smooths over the frames of the chunk.
Same sub-module names as diffusers 0.24 (`decoder.mid_block.resnets.N.spatial_res_block...`, `decoder.time_conv_out`)."""
from __future__ import annotations

from typing import Tuple

import torch
import torch.nn as nn

from . import engine as E
from . import ops
from .autoencoder_kl import AutoencoderKL, DecoderOutput
from .layers import Attention, Upsample2D
from .modeling import capture_config
from .unet_spatio_temporal_condition import SpatioTemporalResBlock, prepare_svd_modules, st_resblock_forward


def _st(cin, cout):
    return SpatioTemporalResBlock(cin, cout, temb_channels=None, eps=1e-6, temporal_eps=1e-5, merge_factor=0.0,
                                  merge_strategy="learned", switch_spatial_to_temporal_mix=True)


class MidBlockTemporalDecoder(nn.Module):
    def __init__(self, in_channels, out_channels, attention_head_dim=512, num_layers=1):
        super().__init__()
        self.resnets = nn.ModuleList([_st(in_channels if i == 0 else out_channels, out_channels) for i in range(num_layers)])
        self.attentions = nn.ModuleList([Attention(in_channels, heads=in_channels // attention_head_dim,
                                                   dim_head=attention_head_dim, bias=True, norm_num_groups=32, eps=1e-6,
                                                   residual_connection=True)])


class UpBlockTemporalDecoder(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers=1, add_upsample=True):
        super().__init__()
        self.resnets = nn.ModuleList([_st(in_channels if i == 0 else out_channels, out_channels) for i in range(num_layers)])
        self.upsamplers = (nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)])
                           if add_upsample else None)


class TemporalDecoder(nn.Module):
    def __init__(self, in_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2):
        super().__init__()
        self.conv_in = nn.Conv2d(in_channels, block_out_channels[-1], 3, padding=1)
        self.mid_block = MidBlockTemporalDecoder(block_out_channels[-1], block_out_channels[-1],
                                                 attention_head_dim=block_out_channels[-1], num_layers=layers_per_block)
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(block_out_channels))
        out_c = rev[0]
        for i in range(len(rev)):
            prev, out_c = out_c, rev[i]
            self.up_blocks.append(UpBlockTemporalDecoder(prev, out_c, num_layers=layers_per_block + 1,
                                                         add_upsample=i != len(rev) - 1))
        self.conv_norm_out = nn.GroupNorm(32, block_out_channels[0], eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, 3, padding=1)
        self.time_conv_out = nn.Conv3d(out_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))


class AutoencoderKLTemporalDecoder(AutoencoderKL):
    def __init__(self, in_channels: int = 3, out_channels: int = 3, down_block_types: Tuple[str] = ("DownEncoderBlock2D",) * 4,
                 block_out_channels: Tuple[int] = (128, 256, 512, 512), layers_per_block: int = 2, latent_channels: int = 4,
                 sample_size: int = 768, scaling_factor: float = 0.18215, force_upcast: bool = True):
        super().__init__(in_channels=in_channels, out_channels=out_channels, down_block_types=down_block_types,
                         block_out_channels=block_out_channels, layers_per_block=layers_per_block,
                         latent_channels=latent_channels, sample_size=sample_size, scaling_factor=scaling_factor,
                         force_upcast=force_upcast)
        capture_config(self, AutoencoderKLTemporalDecoder.__init__, (), dict(
            in_channels=in_channels, out_channels=out_channels, down_block_types=down_block_types,
            block_out_channels=block_out_channels, layers_per_block=layers_per_block, latent_channels=latent_channels,
            sample_size=sample_size, scaling_factor=scaling_factor, force_upcast=force_upcast))
        del self.decoder
        del self.post_quant_conv                      # the temporal-decoder VAE has no post_quant_conv
        self.decoder = TemporalDecoder(latent_channels, out_channels, block_out_channels, layers_per_block)

    def _build_prepared(self, dt, device) -> E.Prepared:
        prep = E.Prepared(dt, device)
        with torch.no_grad():
            prepare_svd_modules(prep, self)
            d = self.decoder
            # conv_out / time_conv_out: 3 output channels padded to 8 so that the frame-axis conv can read them through TMA
            co_w = torch.zeros((8,) + tuple(d.conv_out.weight.shape[1:]), dtype=d.conv_out.weight.dtype, device=device)
            co_w[:3] = d.conv_out.weight.detach()
            co_b = torch.zeros(8, dtype=torch.float32, device=device)
            co_b[:3] = d.conv_out.bias.detach().float()
            tw = torch.zeros((8, 8, 3), dtype=d.time_conv_out.weight.dtype, device=device)
            tw[:3, :3] = d.time_conv_out.weight.detach().reshape(3, 3, 3)
            tb = torch.zeros(8, dtype=torch.float32, device=device)
            tb[:3] = d.time_conv_out.bias.detach().float()
            own = {
                "enc_in": E.prep_conv3x3(self.encoder.conv_in, dt, pad_cin_to=8),
                "enc_norm": E.prep_norm(self.encoder.conv_norm_out),
                "enc_out": E.prep_conv3x3(self.encoder.conv_out, dt),
                "dec_in": E.prep_conv3x3(d.conv_in, dt, pad_cin_to=8),
                "dec_norm": E.prep_norm(d.conv_norm_out),
                "dec_out": (co_w.permute(0, 2, 3, 1).reshape(8, -1).to(dt).contiguous(), co_b),
                "dec_time": (tw.permute(0, 2, 1).reshape(8, 24).to(dt).contiguous(), tb),
                "quant": (self.quant_conv.weight.detach().float().reshape(8, 8).contiguous(),
                          self.quant_conv.bias.detach().float().contiguous()),
            }
            prep.put(self, own)
        return prep

    def _decode_chunk(self, *a, **k):  # the 2-D decoder entry points of the parent do not apply
        raise NotImplementedError("AutoencoderKLTemporalDecoder decodes through decode(z, num_frames)")

    @torch.no_grad()
    def decode(self, z: torch.Tensor, num_frames: int, return_dict: bool = True):
        """diffusers AutoencoderKLTemporalDecoder.decode: z [batch*num_frames, 4, h, w] (already divided by the scaling
        factor) -> sample [batch*num_frames, 3, 8h, 8w] in the model dtype (API-compatibility surface: one permute + cast of
        the kernel output; the pipeline mirror consumes `decode_chunk_video` directly)."""
        vid = self.decode_chunk_video(z, num_frames)
        n = z.shape[0]
        img = vid.permute(0, 2, 1, 3, 4).reshape(n, 3, vid.shape[-2], vid.shape[-1]).to(self.dtype)
        if not return_dict:
            return (img,)
        return DecoderOutput(sample=img)

    @torch.no_grad()
    def decode_chunk_video(self, z: torch.Tensor, num_frames: int) -> torch.Tensor:
        """z [batch*num_frames, 4, h, w] -> fp32 video [batch, 3, num_frames, 8h, 8w] holding the 16-bit-rounded values
        (what `decode(...).sample.float()` gives after the pipeline's reshape/permute, models/pipeline.py:456)."""
        prep = self._prepared()
        own = prep.get(self)
        n, _, hh, ww = z.shape
        if n % num_frames:
            raise ValueError("z.shape[0] must be a multiple of num_frames")
        b = n // num_frames
        g = E.Geo(b, num_frames, hh, ww)
        ctx = E.Ctx(prep, g)
        d = self.decoder
        h = ops.conv3x3(ops.image_to_nhwc8(z.to(prep.dtype)), own["dec_in"][0], own["dec_in"][1])
        h = st_resblock_forward(ctx, d.mid_block.resnets[0], h, g)
        for r, a in zip(d.mid_block.resnets[1:], d.mid_block.attentions):
            h = self._mid_attention(ctx, a, h, g)
            h = st_resblock_forward(ctx, r, h, g)
        for blk in d.up_blocks:
            for r in blk.resnets:
                h = st_resblock_forward(ctx, r, h, g)
            if blk.upsamplers is not None:
                h = E.upsample_forward(ctx, blk.upsamplers[0], h, g)
                g = g.up()
        c0 = d.conv_out.in_channels
        h = ops.groupnorm(h, g.n, g.hw, own["dec_norm"][0], own["dec_norm"][1], 1e-6, True, 32)
        y8 = ops.conv3x3(h.view(g.n, g.h, g.w, c0), own["dec_out"][0], own["dec_out"][1])          # [rows, 8] 16-bit
        y = ops.tconv3(y8, g.b, g.t, g.hw, own["dec_time"][0], own["dec_time"][1], out_f32=True)   # frame-axis conv
        return ops.vae_dec_finalize(y, g.b, g.t, g.h, g.w, prep.dtype == torch.bfloat16)             # [b, 3, f, H, W] fp32

    def decode_video(self, *a, **k):
        raise NotImplementedError("use decode(z, num_frames) (diffusers AutoencoderKLTemporalDecoder surface)")

    decode_frames_uint8 = decode_video
