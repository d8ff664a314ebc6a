"""Mirror of the reference's `models/unet_3d_condition_mask.py` `UNet3DConditionModel`:
same constructor config (:87-110), same sub-module names / state_dict keys (:137-266), same `forward` signature and
semantics (:338-526), executed as a sequence of hand-written sm_90a kernels.

Forward (reference line -> here):
  :376      cat(condition_latent, sample) on the frame axis, T = F + 1      -> fused into `unet_in_assemble`
  :408-420  time_proj / motion_proj / time_embedding, repeat_interleave(T)  -> `_time_embedding` (per batch item; the
            per-resnet `time_emb_proj(silu(emb))` of all 22 resnets is one batched GEMM, applied as a per-sample bias
            in conv1's epilogue instead of a broadcast add)
  :421      encoder_hidden_states.repeat_interleave(T)                      -> not materialised: cross-attention K/V
            are projected once per batch item and shared by its T frames (`kv_batch_div`)
  :424-431  mask repeat + channel cat + permute + conv_in2 / conv_in         -> assemble + implicit-GEMM conv (K padded to 8)
  :437-511  transformer_in, down blocks, mid block, up blocks               -> `run()` of the mirrored block classes
  :514-522  GroupNorm + SiLU + conv_out, reshape, drop frame 0              -> groupnorm + implicit-GEMM (N=4, fp32 out)
            + `unet_out_finalize`
"""
from __future__ import annotations

from typing import Any, Dict, Optional, Tuple, Union

import torch
import torch.nn as nn

from . import engine as E
from . import ops
from .layers import TimestepEmbedding, TransformerTemporalModel, ResnetBlock2D
from .modeling import BaseOutput, ModelBase, capture_config
from .unet_3d_blocks import (CrossAttnDownBlock3D, CrossAttnUpBlock3D, DownBlock3D, UNetMidBlock3DCrossAttn, UpBlock3D,
                             get_down_block, get_up_block)


class UNet3DConditionOutput(BaseOutput):
    pass


class UNet3DConditionModel(ModelBase):
    _supports_gradient_checkpointing = False

    def __init__(
        self,
        sample_size: Optional[int] = None,
        in_channels: int = 4,
        out_channels: int = 4,
        down_block_types: Tuple[str] = ("CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D",
                                        "DownBlock3D"),
        up_block_types: Tuple[str] = ("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D"),
        block_out_channels: Tuple[int] = (320, 640, 1280, 1280),
        layers_per_block: int = 2,
        downsample_padding: int = 1,
        mid_block_scale_factor: float = 1,
        act_fn: str = "silu",
        norm_num_groups: Optional[int] = 32,
        norm_eps: float = 1e-5,
        cross_attention_dim: int = 1024,
        attention_head_dim: Union[int, Tuple[int]] = 64,
        motion_mask=False,
        motion_strength=False,
    ):
        super().__init__()
        capture_config(self, UNet3DConditionModel.__init__, (), dict(
            sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
            down_block_types=down_block_types, up_block_types=up_block_types, block_out_channels=block_out_channels,
            layers_per_block=layers_per_block, downsample_padding=downsample_padding,
            mid_block_scale_factor=mid_block_scale_factor, act_fn=act_fn, norm_num_groups=norm_num_groups,
            norm_eps=norm_eps, cross_attention_dim=cross_attention_dim, attention_head_dim=attention_head_dim,
            motion_mask=motion_mask, motion_strength=motion_strength))
        self.motion_mask = motion_mask
        self.motion_strength = motion_strength
        self.sample_size = sample_size
        if len(down_block_types) != len(up_block_types):
            raise ValueError(f"Must provide the same number of `down_block_types` as `up_block_types`. "
                             f"`down_block_types`: {down_block_types}. `up_block_types`: {up_block_types}.")
        if len(block_out_channels) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `block_out_channels` as `down_block_types`. "
                             f"`block_out_channels`: {block_out_channels}. `down_block_types`: {down_block_types}.")
        if not isinstance(attention_head_dim, int) and len(attention_head_dim) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `attention_head_dim` as `down_block_types`. "
                             f"`attention_head_dim`: {attention_head_dim}. `down_block_types`: {down_block_types}.")
        if act_fn not in ("silu", "swish"):
            raise ValueError("only the reference's act_fn='silu' is implemented")
        if norm_num_groups != 32:
            raise ValueError("only the reference's norm_num_groups=32 is implemented")
        if out_channels != 4 or in_channels != 4:
            raise ValueError("the latent path is specialised for 4 latent channels (SD VAE)")

        c0 = block_out_channels[0]
        self.conv_in = nn.Conv2d(in_channels, c0, kernel_size=3, padding=1)
        self.conv_in2 = nn.Conv2d(5, c0, kernel_size=3, padding=1)
        time_embed_dim = c0 * 4
        self.time_embedding = TimestepEmbedding(c0, time_embed_dim, act_fn=act_fn, cond_proj_dim=c0)
        # constructed by the reference but unused in forward (:157-161,:417) — kept for state_dict compatibility
        self.motion_embedding = nn.Sequential(nn.Linear(c0, time_embed_dim), nn.SiLU(),
                                              nn.Linear(time_embed_dim, time_embed_dim))
        nn.init.zeros_(self.motion_embedding[-1].weight)
        nn.init.zeros_(self.motion_embedding[-1].bias)
        self.transformer_in = TransformerTemporalModel(num_attention_heads=8, attention_head_dim=attention_head_dim
                                                       if isinstance(attention_head_dim, int) else attention_head_dim[0],
                                                       in_channels=c0, num_layers=1)
        self.down_blocks = nn.ModuleList([])
        self.up_blocks = nn.ModuleList([])
        if isinstance(attention_head_dim, int):
            attention_head_dim = (attention_head_dim,) * len(down_block_types)
        output_channel = c0
        for i, down_block_type in enumerate(down_block_types):
            input_channel = output_channel
            output_channel = block_out_channels[i]
            is_final_block = i == len(block_out_channels) - 1
            self.down_blocks.append(get_down_block(
                down_block_type, num_layers=layers_per_block, in_channels=input_channel, out_channels=output_channel,
                temb_channels=time_embed_dim, add_downsample=not is_final_block, resnet_eps=norm_eps,
                resnet_act_fn=act_fn, resnet_groups=norm_num_groups, cross_attention_dim=cross_attention_dim,
                attn_num_head_channels=attention_head_dim[i], downsample_padding=downsample_padding,
                dual_cross_attention=False))
        self.mid_block = UNetMidBlock3DCrossAttn(
            in_channels=block_out_channels[-1], temb_channels=time_embed_dim, resnet_eps=norm_eps,
            resnet_act_fn=act_fn, output_scale_factor=mid_block_scale_factor, cross_attention_dim=cross_attention_dim,
            attn_num_head_channels=attention_head_dim[-1], resnet_groups=norm_num_groups, dual_cross_attention=False)
        self.num_upsamplers = 0
        reversed_block_out_channels = list(reversed(block_out_channels))
        reversed_attention_head_dim = list(reversed(attention_head_dim))
        output_channel = reversed_block_out_channels[0]
        for i, up_block_type in enumerate(up_block_types):
            is_final_block = i == len(block_out_channels) - 1
            prev_output_channel = output_channel
            output_channel = reversed_block_out_channels[i]
            input_channel = reversed_block_out_channels[min(i + 1, len(block_out_channels) - 1)]
            add_upsample = not is_final_block
            if add_upsample:
                self.num_upsamplers += 1
            self.up_blocks.append(get_up_block(
                up_block_type, num_layers=layers_per_block + 1, in_channels=input_channel,
                out_channels=output_channel, prev_output_channel=prev_output_channel, temb_channels=time_embed_dim,
                add_upsample=add_upsample, resnet_eps=norm_eps, resnet_act_fn=act_fn, resnet_groups=norm_num_groups,
                cross_attention_dim=cross_attention_dim, attn_num_head_channels=reversed_attention_head_dim[i],
                dual_cross_attention=False))
        self.conv_norm_out = nn.GroupNorm(num_channels=c0, num_groups=norm_num_groups, eps=norm_eps)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(c0, out_channels, kernel_size=3, padding=1)
        self.__dict__["_aab_prepared"] = None
        self.fuse_geglu = True

    # ------------------------------------------------------------------ diffusers-surface no-ops used by train.py
    def enable_xformers_memory_efficient_attention(self, *a, **k):
        pass

    def set_attention_slice(self, slice_size):
        pass

    def enable_gradient_checkpointing(self):
        raise NotImplementedError("training (backward) is outside the inference hot path (SURVEY.md 8, component 8)")

    # ------------------------------------------------------------------ weight preparation
    def _prepared(self) -> E.Prepared:
        prep = self.__dict__.get("_aab_prepared")
        p0 = self.conv_out.weight
        if prep is not None and prep.dtype == p0.dtype and prep.device == p0.device:
            return prep
        if p0.dtype not in (torch.float16, torch.bfloat16):
            raise TypeError(f"the sm_90a path computes in fp16 or bf16; model dtype is {p0.dtype}. "
                            f"Call .to(torch.float16) / .to(torch.bfloat16). There is no fp32/CPU fallback.")
        if not p0.is_cuda:
            raise RuntimeError("UNet3DConditionModel parameters must live on a CUDA device (no CPU fallback)")
        prep = self._build_prepared(p0.dtype, p0.device)
        self.__dict__["_aab_prepared"] = prep
        return prep

    def _build_prepared(self, dt, device) -> E.Prepared:
        """Kernel-layout copies of every weight (layout conversion only; runs wherever the parameters live)."""
        prep = E.Prepared(dt, device)
        with torch.no_grad():
            E.prepare_module(prep, self)
            own = {}
            own["conv_in"] = E.prep_conv3x3(self.conv_in, dt, pad_cin_to=8)
            own["conv_in2"] = E.prep_conv3x3(self.conv_in2, dt, pad_cin_to=8)
            own["norm_out"] = E.prep_norm(self.conv_norm_out)
            own["conv_out"] = E.prep_conv3x3(self.conv_out, dt)
            # every ResnetBlock2D.time_emb_proj stacked into one [sum(Cout), 1280] matrix
            ws, bs, offs, off = [], [], {}, 0
            for m in self.modules():
                if isinstance(m, ResnetBlock2D) and m.time_emb_proj is not None:
                    offs[id(m)] = off
                    ws.append(m.time_emb_proj.weight.detach())
                    bs.append(m.time_emb_proj.bias.detach())
                    off += m.out_channels
            own["temb_w"] = torch.cat(ws, dim=0).to(dt).contiguous()
            own["temb_b"] = torch.cat(bs, dim=0).float().contiguous()
            own["temb_off"] = offs
            prep.put(self, own)
        return prep

    # ------------------------------------------------------------------ forward
    @staticmethod
    def _check_per_batch(name, count, b, n_shared):
        """The reference broadcasts a [1] or [B] tensor over the batch (:392-406 `timesteps.expand`) and raises on any
        other length; under the shared CFG prefix the caller holds one value per prompt (B = 2 x prompts, batch ordered
        [uncond..., text...]), which tiles over both halves."""
        if count not in (1, b) and not (n_shared and count == n_shared):
            raise ValueError(f"`{name}` has {count} values for a batch of {b}: expected 1 or {b}"
                             + (f" (or {n_shared}, one per prompt)" if n_shared else ""))

    def _time_embedding(self, prep, timestep, motion, b, device, n_shared=0, timestep_cond=None):
        """reference :391-420.  Returns fp32 [B, sum(Cout)] = time_emb_proj_r(silu(emb)) for every resnet r."""
        own = prep.get(self)
        te = prep.get(self.time_embedding)
        dt = prep.dtype
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([float(timestep)], dtype=torch.float32, device=device)
        else:
            timestep = timestep.to(device=device, dtype=torch.float32).reshape(-1)
        self._check_per_batch("timestep", timestep.numel(), b, n_shared)
        c0 = self.conv_in.out_channels
        t_emb = ops.timestep_embed(timestep, b, c0, dt)
        if self.motion_strength and motion is not None:
            if not torch.is_tensor(motion):
                motion = torch.tensor(motion, dtype=torch.float32, device=device)
            motion = motion.to(device=device, dtype=torch.float32).reshape(-1)
            self._check_per_batch("motion", motion.numel(), b, n_shared)
            m_emb = ops.timestep_embed(motion, b, c0, dt)
            t_emb = ops.linear(m_emb, te["cp"], None, residual=t_emb)         # sample + cond_proj(condition)
        elif timestep_cond is not None:
            # :418-419 `self.time_embedding(t_emb, timestep_cond)` when no motion value is in play: [1 | B, C0] broadcast over B
            tc = timestep_cond.to(device=device, dtype=dt).reshape(-1, c0)
            self._check_per_batch("timestep_cond", tc.shape[0], b, n_shared)
            if tc.shape[0] != b:
                tc = tc.repeat(b // tc.shape[0], 1)
            t_emb = ops.linear(tc.contiguous(), te["cp"], None, residual=t_emb)
        h = ops.linear(t_emb, te["l1"][0], te["l1"][1], act=ops.ACT_SILU)
        semb = ops.linear(h, te["l2"][0], te["l2"][1], act=ops.ACT_SILU)      # silu(emb): what every resnet consumes
        return ops.linear(semb, own["temb_w"], own["temb_b"], out_f32=True)

    @torch.no_grad()
    def forward(
        self,
        sample: torch.Tensor,
        timestep: Union[torch.Tensor, float, int],
        encoder_hidden_states: torch.Tensor,
        condition_latent: torch.Tensor,
        mask: torch.Tensor,
        class_labels: Optional[torch.Tensor] = None,
        timestep_cond: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        cross_attention_kwargs: Optional[Dict[str, Any]] = None,
        down_block_additional_residuals: Optional[Tuple[torch.Tensor]] = None,
        mid_block_additional_residual: Optional[torch.Tensor] = None,
        motion=None,
        return_dict: bool = True,
        _raw_eps: bool = False,
        _kv_cache: Optional[dict] = None,
        _cfg_shared_prefix: bool = False,
    ):
        """`_cfg_shared_prefix=True` (used by LatentToVideoPipeline under classifier-free guidance): `sample`,
        `condition_latent` hold ONE copy per prompt ([n, ...]) while `encoder_hidden_states` holds [2n, ...]
        (unconditional first).  Both guidance halves see identical latents / condition / timestep, so every layer before
        the first text cross-attention is evaluated once and duplicated there; the result equals the reference's
        `torch.cat([latents] * 2)` evaluation (models/pipeline.py:165) up to the summation order inside GroupNorm."""
        # `attention_mask` and `class_labels` are accepted and IGNORED, exactly like the reference: its forward turns the
        # mask into a -10000 bias (:385-388) and hands it to blocks whose forward never reads the argument
        # (models/unet_3d_blocks.py:340,489,720), and `class_labels` is never read at all (there is no class embedding).
        # `timestep_cond` feeds `time_embedding.cond_proj` when no motion value is used (:414-419).
        if down_block_additional_residuals is not None or mid_block_additional_residual is not None:
            raise NotImplementedError("ControlNet residuals (:456-479) are not used by any caller in the reference tree and "
                                      "are not implemented")
        if sample.shape[2] + 1 > ops.TEMPORAL_MAX_FRAMES:   # F + 1 frames (condition frame); raise before the first launch
            raise NotImplementedError(f"temporal attention handles up to {ops.TEMPORAL_MAX_FRAMES} frames: {sample.shape[2]} "
                                      f"frames + the condition frame is {sample.shape[2] + 1}")
        prep = self._prepared()
        own = prep.get(self)
        dt = prep.dtype
        dev = prep.device
        if sample.dtype != dt:
            sample = sample.to(dt)
        if condition_latent.dtype != dt:
            condition_latent = condition_latent.to(dt)
        b, c, f, h, w = sample.shape
        b_full = 2 * b if _cfg_shared_prefix else b
        if _cfg_shared_prefix and encoder_hidden_states.shape[0] != b_full:
            raise ValueError("_cfg_shared_prefix needs encoder_hidden_states of batch 2 x sample batch")
        # reference :377-383: when the latent size is not a multiple of 2**num_upsamplers the upsamplers interpolate to
        # the size of the matching skip tensor instead of x2
        forward_upsample_size = any(s % (2 ** self.num_upsamplers) != 0 for s in (h, w))
        g = E.Geo(b, f + 1, h, w)
        ctx = E.Ctx(prep, g)
        ctx.fuse_geglu = self.fuse_geglu
        ctx.temb_off = own["temb_off"]
        ctx.dup_pending = bool(_cfg_shared_prefix)
        ctx.temb_all = self._time_embedding(prep, timestep, motion, b_full, dev, b if _cfg_shared_prefix else 0, timestep_cond)
        ehs = encoder_hidden_states
        if ehs.dtype != dt:
            ehs = ehs.to(dt)
        ctx.lk = ehs.shape[1]
        ctx.ehs = ehs.reshape(-1, ehs.shape[-1]).contiguous()
        if _kv_cache is not None:
            ctx.kv_cache = _kv_cache

        use_mask = bool(self.motion_mask) and mask is not None
        if use_mask and mask.dtype != dt:
            mask = mask.to(dt)
        x8 = ops.unet_in_assemble(sample, condition_latent, mask if use_mask else None, g.t)
        wi = own["conv_in2"] if use_mask else own["conv_in"]
        x = ops.conv3x3(x8.view(g.n, h, w, 8), wi[0], wi[1], stats=True)
        trace = self.__dict__.get("_trace")
        if trace is not None:
            trace.append(("conv_in", x, g))
        if g.t > 1:
            x = E.temporal_transformer_forward(ctx, self.transformer_in, x, g)
            if trace is not None:
                trace.append(("transformer_in", x, g))

        skips = [(x, g)]
        for i, blk in enumerate(self.down_blocks):
            x, g2, outs = blk.run(ctx, x, g)
            skips.extend(outs)
            g = g2
            if trace is not None:
                trace.append((f"down_blocks.{i}", x, g))
        x, g = self.mid_block.run(ctx, x, g)
        if trace is not None:
            trace.append(("mid_block", x, g))
        for i, blk in enumerate(self.up_blocks):
            is_final_block = i == len(self.up_blocks) - 1
            n_res = len(blk.resnets)
            up_size = None
            if not is_final_block and forward_upsample_size:       # reference :486-491: size of the next block's first skip
                sg = skips[-n_res - 1][1]
                up_size = (sg.h, sg.w)
            x, g = blk.run(ctx, x, g, skips, upsample_size=up_size)
            if trace is not None:
                trace.append((f"up_blocks.{i}", x, g))

        if ctx.dup_pending:                       # no cross-attention anywhere: duplicate at the very end
            x = ops.dup_rows(x)
            g = E.Geo(g.b * 2, g.t, g.h, g.w)
            ctx.dup_pending = False
        c0 = self.conv_in.out_channels
        x = ops.groupnorm(x, g.n, g.hw, own["norm_out"][0], own["norm_out"][1], self.conv_norm_out.eps, True, 32)
        eps = ops.conv3x3(x.view(g.n, g.h, g.w, c0), own["conv_out"][0], own["conv_out"][1], out_f32=True)
        if _raw_eps:
            return eps, g            # fp32 [B*T*h*w, 4] channels-last, consumed by the fused CFG+scheduler kernel
        out = ops.unet_out_finalize(eps, b_full, g.t, h, w, dt)
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)
