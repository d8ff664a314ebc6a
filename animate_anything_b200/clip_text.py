"""Mirror of `transformers.CLIPTextModel` as the reference uses it: `LatentToVideoPipeline._encode_prompt`
(models/pipeline.py:136 -> diffusers TextToVideoSDPipeline._encode_prompt) calls
`self.text_encoder(text_input_ids.to(device), attention_mask=None)[0]` on the model loaded at train.py:88
(`CLIPTextModel.from_pretrained(path, subfolder="text_encoder")`), cast to fp16 on the GPU at train.py:851.

Same sub-module names (-> identical state_dict keys: `text_model.embeddings.token_embedding.weight`,
`text_model.encoder.layers.N.self_attn.{q,k,v,out}_proj`, `layer_norm1/2`, `mlp.fc1/fc2`, `text_model.final_layer_norm`),
same call signature and outputs (`[0]` = last_hidden_state [B, L, C], `.pooler_output` = the EOS-token row).

Execution (all through the C-ABI, no library GEMM / SDPA):
  token + position embedding   -> `aab_embed_tokens`
  per layer: LayerNorm -> fused q|k|v Linear (one [3C, C] wgmma GEMM, bias in the epilogue) -> causal head-dim-64 flash
             attention (`aab_flash_attn_d64`, causal bit) -> out_proj (+ residual in the epilogue) -> LayerNorm ->
             fc1 (+ GELU / quick-GELU) -> fc2 (+ residual)
  final LayerNorm; pooled row gathered with `aab_copy2d`.
The parity oracle for this file is the REAL third-party implementation: `transformers` is installed in the image
(tests/test_gpu_clip.py), so this leg is pinned to the library the reference imports, not to a restatement.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import _lib, ops
from .modeling import BaseOutput, ModelBase, capture_config


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
    def __init__(self, vocab, c, max_pos):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab, c)
        self.position_embedding = nn.Embedding(max_pos, c)


class _Encoder(nn.Module):
    def __init__(self, n, c, inner, eps):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(c, inner, eps) for _ in range(n)])


class _TextTransformer(nn.Module):
    def __init__(self, vocab, c, inner, n, max_pos, eps):
        super().__init__()
        self.embeddings = _Embeddings(vocab, c, max_pos)
        self.encoder = _Encoder(n, c, inner, eps)
        self.final_layer_norm = nn.LayerNorm(c, eps=eps)


class CLIPTextModelOutput(BaseOutput):
    pass


class CLIPTextModel(ModelBase):
    config_name = "config.json"
    weights_name = "model"                 # transformers: model.safetensors / pytorch_model.bin
    weights_bin_name = "pytorch_model.bin"

    def __init__(self, vocab_size: int = 49408, hidden_size: int = 1024, intermediate_size: int = 4096,
                 num_hidden_layers: int = 23, num_attention_heads: int = 16, max_position_embeddings: int = 77,
                 hidden_act: str = "gelu", layer_norm_eps: float = 1e-5, eos_token_id: int = 49407,
                 projection_dim: int = 512, pad_token_id: int = 1, bos_token_id: int = 49406):
        super().__init__()
        capture_config(self, CLIPTextModel.__init__, (), dict(
            vocab_size=vocab_size, hidden_size=hidden_size, intermediate_size=intermediate_size,
            num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
            max_position_embeddings=max_position_embeddings, hidden_act=hidden_act, layer_norm_eps=layer_norm_eps,
            eos_token_id=eos_token_id, projection_dim=projection_dim, pad_token_id=pad_token_id,
            bos_token_id=bos_token_id))
        if hidden_size != 64 * num_attention_heads:
            raise ValueError("the sm_90a attention kernel is specialised for head_dim 64 (ViT-H/14 and ViT-L/14 text towers)")
        if hidden_act not in ("gelu", "quick_gelu"):
            raise ValueError(f"hidden_act {hidden_act!r} is not a CLIP text activation")
        if max_position_embeddings > 128:
            raise ValueError("causal attention kernel handles up to 128 tokens (CLIP: 77)")
        self.text_model = _TextTransformer(vocab_size, hidden_size, intermediate_size, num_hidden_layers,
                                           max_position_embeddings, layer_norm_eps)
        self.__dict__["_aab_prepared"] = None

    # ------------------------------------------------------------------ construction from the library model
    @classmethod
    def from_hf(cls, hf_model) -> "CLIPTextModel":
        """Mirror of an instantiated `transformers.CLIPTextModel` (what train.py:88 creates): same config, same weights,
        same dtype/device."""
        c = hf_model.config
        m = cls(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
                max_position_embeddings=c.max_position_embeddings, hidden_act=c.hidden_act,
                layer_norm_eps=c.layer_norm_eps, eos_token_id=c.eos_token_id,
                projection_dim=getattr(c, "projection_dim", 512))
        p0 = next(hf_model.parameters())
        m = m.to(device=p0.device, dtype=p0.dtype)
        m.load_state_dict(hf_model.state_dict())
        return m.eval()

    def _convert_legacy_keys(self, sd):
        return {k: v for k, v in sd.items() if not k.endswith("position_ids")}

    def load_state_dict(self, sd, strict=True, **kw):
        return super().load_state_dict(self._convert_legacy_keys(sd), strict=strict, **kw)

    # ------------------------------------------------------------------ weights
    def _prepared(self) -> dict:
        prep = self.__dict__.get("_aab_prepared")
        p0 = self.text_model.final_layer_norm.weight
        if prep is not None and prep["dtype"] == p0.dtype and prep["device"] == p0.device:
            return prep
        if p0.dtype not in (torch.float16, torch.bfloat16) or not p0.is_cuda:
            raise TypeError("CLIPTextModel must be fp16/bf16 on a CUDA device for the sm_90a path (train.py:851 casts "
                            "it to half on cuda); there is no library / CPU fallback")
        dt = p0.dtype
        f32 = lambda t: t.detach().float().contiguous()
        w = lambda t: t.detach().to(dt).contiguous()
        tm = self.text_model
        layers = []
        with torch.no_grad():
            for ly in tm.encoder.layers:
                a = ly.self_attn
                layers.append(dict(
                    n1=(f32(ly.layer_norm1.weight), f32(ly.layer_norm1.bias)),
                    qkv=w(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], dim=0)),
                    qkv_b=f32(torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], dim=0)),
                    o=(w(a.out_proj.weight), f32(a.out_proj.bias)),
                    n2=(f32(ly.layer_norm2.weight), f32(ly.layer_norm2.bias)),
                    fc1=(w(ly.mlp.fc1.weight), f32(ly.mlp.fc1.bias)),
                    fc2=(w(ly.mlp.fc2.weight), f32(ly.mlp.fc2.bias))))
            prep = dict(dtype=dt, device=p0.device, layers=layers,
                        tok=w(tm.embeddings.token_embedding.weight), pos=w(tm.embeddings.position_embedding.weight),
                        nf=(f32(tm.final_layer_norm.weight), f32(tm.final_layer_norm.bias)))
        self.__dict__["_aab_prepared"] = prep
        return prep

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, position_ids=None,
                output_attentions=None, output_hidden_states=None, return_dict=None):
        """transformers CLIPTextModel.forward / CLIPTextTransformer.forward: causal self-attention over the tokens."""
        if attention_mask is not None and not bool(attention_mask.bool().all()):
            raise NotImplementedError("padding attention_mask is not used by the reference (CLIP configs have no "
                                      "`use_attention_mask`; models/pipeline.py:136 passes None)")
        if position_ids is not None or output_attentions or output_hidden_states:
            raise NotImplementedError("position_ids / output_attentions / output_hidden_states are not used by the reference")
        prep = self._prepared()
        cfg = self.config
        b, l = input_ids.shape
        if l > cfg.max_position_embeddings:
            raise ValueError(f"sequence length {l} exceeds max_position_embeddings {cfg.max_position_embeddings}")
        c = cfg.hidden_size
        heads = cfg.num_attention_heads
        ids = input_ids.to(device=prep["device"], dtype=torch.int64).contiguous()
        act = ops.ACT_GELU if cfg.hidden_act == "gelu" else ops.ACT_QUICK_GELU
        eps = cfg.layer_norm_eps
        hs = ops.embed_tokens(ids.view(-1), prep["tok"], prep["pos"], l)                # [b*l, c]
        for p in prep["layers"]:
            n1 = ops.layernorm(hs, p["n1"][0], p["n1"][1], eps)
            qkv = ops.linear(n1, p["qkv"], p["qkv_b"])                                   # [b*l, 3c]
            a = ops.flash_attn_d64(qkv, 0, qkv, c, 2 * c, b, l, l, heads, causal=True)
            hs = ops.linear(a, p["o"][0], p["o"][1], residual=hs)
            n2 = ops.layernorm(hs, p["n2"][0], p["n2"][1], eps)
            f = ops.linear(n2, p["fc1"][0], p["fc1"][1], act=act)
            hs = ops.linear(f, p["fc2"][0], p["fc2"][1], residual=hs)
        last = ops.layernorm(hs, prep["nf"][0], prep["nf"][1], eps).view(b, l, c)
        # pooled output: the row of the EOS token (transformers: argmax of the ids when eos_token_id == 2, else the first
        # position equal to eos_token_id).  Index arithmetic on the host-visible ids; the row copy is a C-ABI kernel.
        if cfg.eos_token_id == 2:
            pos = ids.to(torch.int32).argmax(dim=-1)
        else:
            pos = (ids.to(torch.int32) == cfg.eos_token_id).int().argmax(dim=-1)
        pooled = torch.empty((b, c), device=last.device, dtype=last.dtype)
        flat = last.view(b * l, c)
        for i, pidx in enumerate(pos.tolist()):
            _lib.call("aab_copy2d", ops._ptr(flat[i * l + pidx]), c, ops._ptr(pooled[i]), c, 1, c, ops._stream())
        if return_dict is False:
            return (last, pooled)
        return CLIPTextModelOutput(last_hidden_state=last, pooler_output=pooled)
