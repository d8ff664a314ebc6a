"""Mirror of `transformers.CLIPVisionModelWithProjection` as the SVD pipelines use it: `_encode_image` of
`MaskStableVideoDiffusionPipeline` / `TextStableVideoDiffusionPipeline` (models/pipeline.py:347,597 -> diffusers 0.24
StableVideoDiffusionPipeline._encode_image) calls `self.image_encoder(image).image_embeds` on the ViT-H/14 image tower the
pipeline was loaded with (`image_encoder/`: 32 layers, width 1280, 16 heads of 80, 224 px, patch 14, projection 1024).

Same sub-module names (-> identical state_dict keys: `vision_model.embeddings.{class_embedding, patch_embedding.weight,
position_embedding.weight}`, `vision_model.pre_layrnorm`, `vision_model.encoder.layers.N.self_attn.{q,k,v,out}_proj`,
`layer_norm1/2`, `mlp.fc1/fc2`, `vision_model.post_layernorm`, `visual_projection.weight`), same outputs (`image_embeds`
[B, projection_dim], `last_hidden_state` [B, 257, C] before `post_layernorm`).

Execution (all through the C-ABI, no library GEMM / SDPA / conv):
  image -> patch matrix        -> `aab_clip_image_prep` (PIL uint8: diffusers' resize + CLIP normalisation; tensors: rounding)
  patch embedding              -> one wgmma GEMM over [B * 257, 592] (row 0 of each image is a zero patch: the class slot)
  class + position embedding   -> `aab_add_rowvec` with a position table whose row 0 has `class_embedding` added
  pre_layrnorm, 32 x (LayerNorm -> fused q|k|v GEMM -> head-dim-80 flash attention (`aab_flash_attn_d80`) -> out_proj
  (+ residual) -> LayerNorm -> fc1 (+ GELU) -> fc2 (+ residual)), post_layernorm on token 0 of each image (a strided
  LayerNorm, no gather), visual_projection.
The parity oracle for this file is the real `transformers` implementation (tests/test_gpu_clip_vision.py).

The host-side constants of diffusers' image path (`_resize_with_antialiasing`: sigma, kernel size, Gaussian taps; the
order /255 -> [-1, 1] -> blur -> bicubic -> [0, 1] -> normalise) are recalled from diffusers 0.24, which is not vendored
here: parity unpinned, like the rest of the diffusers shim.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .modeling import BaseOutput, ModelBase, capture_config

# transformers.image_utils OPENAI_CLIP_MEAN / OPENAI_CLIP_STD (CLIPImageProcessor defaults)
OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def antialias_params(h: int, w: int, size=(224, 224)):
    """diffusers `_resize_with_antialiasing` (parity unpinned): per axis factor = size_in / size_out,
    sigma = max((factor - 1) / 2, 0.001), kernel size = int(max(2 * 2 * sigma, 3)) bumped to odd.
    Returns ((ks_y, sigma_y), (ks_x, sigma_x))."""
    out = []
    for n, s in ((h, size[0]), (w, size[1])):
        sigma = max((n / s - 1.0) / 2.0, 0.001)
        ks = int(max(2.0 * 2 * sigma, 3))
        if ks % 2 == 0:
            ks += 1
        out.append((ks, sigma))
    return tuple(out)


def gaussian_taps(ks: int, sigma: float) -> torch.Tensor:
    """diffusers `_gaussian` in fp32 on the host, exactly as torch computes it: exp(-x^2 / (2 sigma^2)) over
    x = arange(ks) - ks // 2, normalised to sum 1."""
    sig = torch.tensor([[sigma]], dtype=torch.float32)
    x = (torch.arange(ks, dtype=torch.float32) - ks // 2).expand(1, -1)
    if ks % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2 * sig.pow(2.0)))
    return (g / g.sum(-1, keepdim=True))[0].contiguous()


class _Attn(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.k_proj = nn.Linear(c, c)
        self.v_proj = nn.Linear(c, c)
        self.q_proj = nn.Linear(c, c)
        self.out_proj = nn.Linear(c, c)


class _MLP(nn.Module):
    def __init__(self, c, inner):
        super().__init__()
        self.fc1 = nn.Linear(c, inner)
        self.fc2 = nn.Linear(inner, c)


class _Layer(nn.Module):
    def __init__(self, c, inner, eps):
        super().__init__()
        self.self_attn = _Attn(c)
        self.layer_norm1 = nn.LayerNorm(c, eps=eps)
        self.mlp = _MLP(c, inner)
        self.layer_norm2 = nn.LayerNorm(c, eps=eps)


class _Embeddings(nn.Module):
    def __init__(self, c, channels, image_size, patch):
        super().__init__()
        self.class_embedding = nn.Parameter(torch.randn(c))
        self.patch_embedding = nn.Conv2d(channels, c, kernel_size=patch, stride=patch, bias=False)
        self.position_embedding = nn.Embedding((image_size // patch) ** 2 + 1, c)


class _Encoder(nn.Module):
    def __init__(self, n, c, inner, eps):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(c, inner, eps) for _ in range(n)])


class _VisionTransformer(nn.Module):
    def __init__(self, c, inner, n, channels, image_size, patch, eps):
        super().__init__()
        self.embeddings = _Embeddings(c, channels, image_size, patch)
        self.pre_layrnorm = nn.LayerNorm(c, eps=eps)
        self.encoder = _Encoder(n, c, inner, eps)
        self.post_layernorm = nn.LayerNorm(c, eps=eps)


class CLIPVisionModelOutput(BaseOutput):
    pass


class CLIPVisionModelWithProjection(ModelBase):
    config_name = "config.json"
    weights_name = "model"                 # transformers: model.safetensors / pytorch_model.bin
    weights_bin_name = "pytorch_model.bin"

    def __init__(self, hidden_size: int = 1280, intermediate_size: int = 5120, projection_dim: int = 1024,
                 num_hidden_layers: int = 32, num_attention_heads: int = 16, num_channels: int = 3, image_size: int = 224,
                 patch_size: int = 14, hidden_act: str = "gelu", layer_norm_eps: float = 1e-5):
        super().__init__()
        capture_config(self, CLIPVisionModelWithProjection.__init__, (), dict(
            hidden_size=hidden_size, intermediate_size=intermediate_size, projection_dim=projection_dim,
            num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads, num_channels=num_channels,
            image_size=image_size, patch_size=patch_size, hidden_act=hidden_act, layer_norm_eps=layer_norm_eps))
        if hidden_size != 80 * num_attention_heads:
            raise ValueError("the sm_90a vision attention kernel is specialised for head_dim 80 (ViT-H/14 image tower), got "
                             f"{hidden_size} / {num_attention_heads}")
        if hidden_act not in ("gelu", "quick_gelu"):
            raise ValueError(f"hidden_act {hidden_act!r} is not a CLIP activation")
        if num_channels != 3 or image_size % patch_size:
            raise ValueError("CLIP image towers take 3-channel images whose size is a multiple of the patch size")
        self.vision_model = _VisionTransformer(hidden_size, intermediate_size, num_hidden_layers, num_channels, image_size,
                                               patch_size, layer_norm_eps)
        self.visual_projection = nn.Linear(hidden_size, projection_dim, bias=False)
        self.__dict__["_aab_prepared"] = None

    @property
    def k_pad(self) -> int:
        """Width of the patch-embedding GEMM's K: 3 * patch^2 rounded up to 8 (16-byte rows; 588 -> 592)."""
        k = 3 * self.config.patch_size ** 2
        return -(-k // 8) * 8

    # ------------------------------------------------------------------ construction from the library model
    @classmethod
    def from_hf(cls, hf_model) -> "CLIPVisionModelWithProjection":
        """Mirror of an instantiated `transformers.CLIPVisionModelWithProjection`: same config, weights, dtype, device."""
        c = hf_model.config
        m = cls(hidden_size=c.hidden_size, intermediate_size=c.intermediate_size, projection_dim=c.projection_dim,
                num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
                num_channels=c.num_channels, image_size=c.image_size, patch_size=c.patch_size, hidden_act=c.hidden_act,
                layer_norm_eps=c.layer_norm_eps)
        p0 = next(hf_model.parameters())
        m = m.to(device=p0.device, dtype=p0.dtype)
        m.load_state_dict(hf_model.state_dict())
        return m.eval()

    def _convert_legacy_keys(self, sd):
        return {k: v for k, v in sd.items() if not k.endswith("position_ids")}

    def load_state_dict(self, sd, strict=True, **kw):
        return super().load_state_dict(self._convert_legacy_keys(sd), strict=strict, **kw)

    # ------------------------------------------------------------------ weights
    def _build_prepared(self, dt, device) -> dict:
        """Kernel-layout weights: fused q|k|v, fp32 biases / norms, the patch weight [C, k_pad] zero-padded, the fp32
        position table [257, C] with `class_embedding` added to row 0."""
        f32 = lambda t: t.detach().float().contiguous()
        w = lambda t: t.detach().to(dt).contiguous()
        vm = self.vision_model
        emb = vm.embeddings
        layers = []
        with torch.no_grad():
            for ly in vm.encoder.layers:
                a = ly.self_attn
                layers.append(dict(
                    n1=(f32(ly.layer_norm1.weight), f32(ly.layer_norm1.bias)),
                    qkv=w(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], dim=0)),
                    qkv_b=f32(torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], dim=0)),
                    o=(w(a.out_proj.weight), f32(a.out_proj.bias)),
                    n2=(f32(ly.layer_norm2.weight), f32(ly.layer_norm2.bias)),
                    fc1=(w(ly.mlp.fc1.weight), f32(ly.mlp.fc1.bias)),
                    fc2=(w(ly.mlp.fc2.weight), f32(ly.mlp.fc2.bias))))
            pw = emb.patch_embedding.weight.detach().to(dt).flatten(1)
            patch_w = torch.zeros((pw.shape[0], self.k_pad), dtype=dt, device=pw.device)
            patch_w[:, :pw.shape[1]] = pw
            # the 16-bit model adds 16-bit class / position values: the fp32 sum of the two 16-bit values, rounded once
            pos = emb.position_embedding.weight.detach().to(dt).float().clone()
            pos[0] += emb.class_embedding.detach().to(dt).float()
            prep = dict(dtype=dt, device=device, layers=layers, patch_w=patch_w.contiguous(), pos=pos.contiguous(),
                        pre=(f32(vm.pre_layrnorm.weight), f32(vm.pre_layrnorm.bias)),
                        post=(f32(vm.post_layernorm.weight), f32(vm.post_layernorm.bias)),
                        proj=w(self.visual_projection.weight))
        return prep

    def _prepared(self) -> dict:
        prep = self.__dict__.get("_aab_prepared")
        p0 = self.vision_model.post_layernorm.weight
        if prep is not None and prep["dtype"] == p0.dtype and prep["device"] == p0.device:
            return prep
        if p0.dtype not in (torch.float16, torch.bfloat16) or not p0.is_cuda:
            raise TypeError("CLIPVisionModelWithProjection must be fp16/bf16 on a CUDA device for the sm_90a path; there is "
                            "no library / CPU fallback")
        prep = self._build_prepared(p0.dtype, p0.device)
        self.__dict__["_aab_prepared"] = prep
        return prep

    # ------------------------------------------------------------------ forward
    def _tower(self, prep: dict, x: torch.Tensor, b: int):
        """x: the patch matrix [b * (1 + n_patches), k_pad] from `ops.clip_image_prep`."""
        cfg = self.config
        c, heads, eps = cfg.hidden_size, cfg.num_attention_heads, cfg.layer_norm_eps
        l = (cfg.image_size // cfg.patch_size) ** 2 + 1
        act = ops.ACT_GELU if cfg.hidden_act == "gelu" else ops.ACT_QUICK_GELU
        hs = ops.linear(x, prep["patch_w"])                                         # [b*l, c]; class rows are zeros
        hs = ops.add_rowvec(hs, prep["pos"], 1, l, inplace=True)                   # + class / position embedding
        hs = ops.layernorm(hs, prep["pre"][0], prep["pre"][1], eps)
        for p in prep["layers"]:
            n1 = ops.layernorm(hs, p["n1"][0], p["n1"][1], eps)
            qkv = ops.linear(n1, p["qkv"], p["qkv_b"])                              # [b*l, 3c]
            a = ops.flash_attn_d80(qkv, 0, qkv, c, 2 * c, b, l, l, heads)
            hs = ops.linear(a, p["o"][0], p["o"][1], residual=hs)
            n2 = ops.layernorm(hs, p["n2"][0], p["n2"][1], eps)
            f = ops.linear(n2, p["fc1"][0], p["fc1"][1], act=act)
            hs = ops.linear(f, p["fc2"][0], p["fc2"][1], residual=hs)
        last = hs.view(b, l, c)
        pooled = ops.layernorm(last[:, 0], prep["post"][0], prep["post"][1], eps)  # token 0 rows, stride l*c
        emb = ops.linear(pooled, prep["proj"])
        return CLIPVisionModelOutput(image_embeds=emb, last_hidden_state=last)

    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor, interpolate_pos_encoding: bool = False, output_attentions=None,
                output_hidden_states=None, return_dict=None):
        """transformers CLIPVisionModelWithProjection.forward on CLIP pixel values [B, 3, S, S] (any float dtype)."""
        if interpolate_pos_encoding or output_attentions or output_hidden_states:
            raise NotImplementedError("interpolate_pos_encoding / output_attentions / output_hidden_states are not used by "
                                      "the SVD pipelines")
        cfg = self.config
        if pixel_values.dim() != 4:
            raise ValueError(f"pixel_values must be [B, C, H, W], got {tuple(pixel_values.shape)}")
        h, w = pixel_values.shape[-2:]
        if h != cfg.image_size or w != cfg.image_size:
            raise ValueError(f"Input image size ({h}*{w}) doesn't match model ({cfg.image_size}*{cfg.image_size}).")
        prep = self._prepared()
        pv = pixel_values
        if pv.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            if pv.is_cuda:
                raise TypeError(f"pixel_values must be float32 / float16 / bfloat16, got {pv.dtype}")
            pv = pv.float()                                                         # host conversion, before the upload
        pv = pv.to(prep["device"])
        x = ops.clip_image_prep(pv, prep["dtype"], cfg.image_size, cfg.patch_size, self.k_pad)
        out = self._tower(prep, x, pv.shape[0])
        if return_dict is False:
            return (out.image_embeds, out.last_hidden_state)
        return out

    @torch.no_grad()
    def encode_images(self, images_u8: torch.Tensor, image_mean=OPENAI_CLIP_MEAN, image_std=OPENAI_CLIP_STD):
        """diffusers 0.24 `_encode_image` for PIL input, from the uint8 pixels [B, H, W, 3] (`np.array(pil_image)`): resize
        with antialiasing to the model's size, CLIP normalisation, then the tower -- the preprocessing on the GPU in one
        kernel.  The blur taps are computed on the host, as torch computes them."""
        if images_u8.dtype != torch.uint8 or images_u8.dim() != 4 or images_u8.shape[-1] != 3:
            raise ValueError(f"expected uint8 RGB images [B, H, W, 3], got {images_u8.dtype} {tuple(images_u8.shape)}")
        cfg = self.config
        prep = self._prepared()
        dev = prep["device"]
        h, w = images_u8.shape[1:3]
        (ks_y, sig_y), (ks_x, sig_x) = antialias_params(h, w, (cfg.image_size, cfg.image_size))
        taps_y = gaussian_taps(ks_y, sig_y).to(dev)
        taps_x = gaussian_taps(ks_x, sig_x).to(dev)
        mean_std = torch.tensor(list(image_mean) + list(image_std), dtype=torch.float32).to(dev)
        u8 = images_u8.to(dev)
        x = ops.clip_image_prep(u8, prep["dtype"], cfg.image_size, cfg.patch_size, self.k_pad, taps_y, taps_x, mean_std)
        return self._tower(prep, x, u8.shape[0])
