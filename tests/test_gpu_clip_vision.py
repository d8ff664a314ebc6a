"""GPU: the CLIP image path of the SVD pipelines on the sm_90a kernels.  `aab_flash_attn_d80` against fp32 softmax attention
on the same 16-bit inputs; `aab_clip_image_prep` against the CPU restatement of diffusers' preprocessing
(tests/clip_vision_emulation.py, pinned by tests/test_clip_vision_cpu.py); the whole tower against the REAL
`transformers.CLIPVisionModelWithProjection`; both SVD pipelines with a transformers image encoder and a PIL image."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import clip_vision_emulation as cve  # noqa: E402
from test_clip_vision_cpu import hf_vision  # noqa: E402
from test_gpu_attention import TOL, _rand, _ref_attn  # noqa: E402
from util import assert_vs_stock, check, record_parity  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nb,l", [(1, 1), (3, 65), (2, 257), (1, 1024)])
def test_flash_d80_self(dtype, nb, l):
    from animate_anything_b200 import ops
    heads = 16
    c = heads * 80
    qkv = _rand((nb * l, 3 * c), dtype, 1.0, 1)
    out = ops.flash_attn_d80(qkv, 0, qkv, c, 2 * c, nb, l, l, heads)
    torch.cuda.synchronize()
    t = qkv.reshape(nb, l, 3, heads, 80).permute(2, 0, 3, 1, 4)
    ref = _ref_attn(t[0], t[1], t[2], 80 ** -0.5).permute(0, 2, 1, 3).reshape(nb * l, c)
    check(f"flash d80 self nb{nb} l{l} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_flash_d80_cross(dtype):
    """Lq != Lk (ragged in both), K/V shared by `kv_batch_div` consecutive query batches."""
    from animate_anything_b200 import ops
    b, t, lq, lk, heads = 2, 3, 150, 77, 16
    c = heads * 80
    q = _rand((b * t * lq, c), dtype, 1.0, 1)
    kv = _rand((b * lk, 2 * c), dtype, 1.0, 2)
    out = ops.flash_attn_d80(q, 0, kv, 0, c, b * t, lq, lk, heads, kv_batch_div=t)
    torch.cuda.synchronize()
    qq = q.reshape(b * t, lq, heads, 80).permute(0, 2, 1, 3)
    kk = kv[:, :c].reshape(b, 1, lk, heads, 80).expand(b, t, lk, heads, 80).reshape(b * t, lk, heads, 80).permute(0, 2, 1, 3)
    vv = kv[:, c:].reshape(b, 1, lk, heads, 80).expand(b, t, lk, heads, 80).reshape(b * t, lk, heads, 80).permute(0, 2, 1, 3)
    ref = _ref_attn(qq, kk, vv, 80 ** -0.5).permute(0, 2, 1, 3).reshape(b * t * lq, c)
    check(f"flash d80 cross {dtype}", out, ref, *TOL[dtype])


def _u8(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (b, h, w, 3), generator=g, dtype=torch.uint8)


def _ulps(got, want, dtype):
    """Distance in units of the 16-bit type's last place (elementwise, via the integer representation)."""
    gi = got.view(torch.int16).int()
    wi = want.view(torch.int16).int()
    gi = torch.where(gi < 0, -32768 - gi, gi)         # sign-magnitude -> monotone integers
    wi = torch.where(wi < 0, -32768 - wi, wi)
    return (gi - wi).abs()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("b,h,w", [(1, 576, 1024), (1, 333, 577), (1, 80, 100), (2, 224, 300)])
def test_clip_image_prep_matches_restatement(dtype, b, h, w):
    from animate_anything_b200 import ops
    from animate_anything_b200.clip_vision import OPENAI_CLIP_MEAN, OPENAI_CLIP_STD, antialias_params, gaussian_taps
    u8 = _u8(b, h, w, seed=h + w)
    (ky, sy), (kx, sx) = antialias_params(h, w)
    ms = torch.tensor(OPENAI_CLIP_MEAN + OPENAI_CLIP_STD, dtype=torch.float32).cuda()
    got = ops.clip_image_prep(u8.cuda(), dtype, 224, 14, 592, gaussian_taps(ky, sy).cuda(), gaussian_taps(kx, sx).cuda(), ms)
    torch.cuda.synchronize()
    want = cve.patch_matrix(cve.preprocess_u8(u8), dtype, 14, 592)
    u = _ulps(got.cpu(), want, dtype)
    assert u.max().item() <= 1, (u.max().item(), (u > 0).float().mean().item())
    # float sources: rounding only
    pv = torch.randn(b, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    for src in (pv, pv.to(dtype), pv.to(torch.bfloat16 if dtype == torch.float16 else torch.float16)):
        got = ops.clip_image_prep(src.cuda(), dtype, 224, 14, 592)
        assert torch.equal(got.cpu(), cve.patch_matrix(src, dtype, 14, 592))


def _tower_case(dtype, act, over, seed, b=2):
    from animate_anything_b200.clip_vision import CLIPVisionModelWithProjection
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    hf = hf_vision(seed=seed, act=act, **over)
    sd16 = {k: v.to(dtype) for k, v in hf.state_dict().items()}
    hf.load_state_dict({k: v.float() for k, v in sd16.items()})
    ours = CLIPVisionModelWithProjection.from_hf(hf).to(dtype).cuda()
    hf = hf.cuda()
    pv = torch.randn(b, 3, 224, 224, generator=torch.Generator().manual_seed(seed + 1)).to(dtype).cuda()
    with torch.no_grad():
        ref = hf(pixel_values=pv.float())
        stock = hf.to(dtype)(pixel_values=pv)
    out = ours(pv)
    torch.cuda.synchronize()
    name = f"CLIP vision {hf.config.num_hidden_layers}L x {hf.config.hidden_size} {str(dtype).split('.')[-1]} {act}"
    assert_vs_stock(record_parity(name, "image_embeds", out.image_embeds, ref.image_embeds, stock.image_embeds),
                    max_factor=2.5)
    assert_vs_stock(record_parity(name, "last_hidden_state", out.last_hidden_state, ref.last_hidden_state,
                                  stock.last_hidden_state), max_factor=2.5)


@pytest.mark.parametrize("dtype,act", [(torch.float16, "gelu"), (torch.bfloat16, "quick_gelu")])
def test_clip_vision_small_matches_transformers(dtype, act):
    _tower_case(dtype, act, {}, seed=0)


def test_clip_vision_vit_h14_full_size_matches_transformers():
    """The SVD image encoder's size: 32 layers x 1280, 16 heads of 80, 224 px, projection 1024 (random weights)."""
    _tower_case(torch.float16, "gelu", dict(hidden_size=1280, intermediate_size=5120, projection_dim=1024,
                                             num_hidden_layers=32, num_attention_heads=16), seed=5, b=1)


# ---------------------------------------------------------------------------------------------- pipelines
def _diffusers_embedding(hf, fe, pil):
    """diffusers 0.24 `_encode_image` for a PIL image, in fp32: the restated preprocessing, then the library tower."""
    u8 = torch.from_numpy(np.array(pil))[None]
    pv = cve.preprocess_u8(u8, 224, fe.image_mean, fe.image_std)
    with torch.no_grad():
        return hf.float()(pixel_values=pv.cuda()).image_embeds


@pytest.mark.parametrize("which", ["mask", "text"])
def test_svd_pipelines_encode_pil_images_on_the_kernels(which, monkeypatch):
    import PIL.Image
    from transformers import CLIPImageProcessor
    from oracle.composition import SVD_SCHED
    from animate_anything_b200.clip_vision import CLIPVisionModelWithProjection
    from animate_anything_b200.pipeline_svd import MaskStableVideoDiffusionPipeline, TextStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from test_gpu_svd import _pair, _vae_pair
    torch.backends.cuda.matmul.allow_tf32 = False
    dtype = torch.float16
    _, unet = _pair(dtype)
    _, vae = _vae_pair(dtype)
    hf = hf_vision(seed=3)
    sd16 = {k: v.to(dtype) for k, v in hf.state_dict().items()}
    hf.load_state_dict({k: v.float() for k, v in sd16.items()})
    fe = CLIPImageProcessor(image_mean=[0.5, 0.45, 0.4], image_std=[0.25, 0.3, 0.27])
    pil = PIL.Image.fromarray(_u8(1, 128, 192, seed=9)[0].numpy())
    want = _diffusers_embedding(hf.cuda(), fe, pil)
    with torch.no_grad():
        stock = hf.to(dtype)(pixel_values=cve.preprocess_u8(torch.from_numpy(np.array(pil))[None], 224, fe.image_mean,
                                                              fe.image_std).to(dtype).cuda()).image_embeds
    cls = MaskStableVideoDiffusionPipeline if which == "mask" else TextStableVideoDiffusionPipeline
    pipe = cls(vae=vae, image_encoder=hf, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED), feature_extractor=fe)

    def boom(*a, **k):
        raise AssertionError("library CLIP vision forward was called")
    monkeypatch.setattr(type(hf), "forward", boom)
    # the embedding: no library conv / GEMM / SDPA kernel on the device during _encode_image
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        emb = pipe._encode_image(None, torch.device("cuda"), 1, True, raw_image=pil)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    library_kernel = lambda n: "aab::" not in n and any(k in n.lower() for k in ("gemm", "sdpa", "flash_fwd", "cudnn",
                                                                                   "fmha", "conv"))
    bad = [n for n in names if n in ("aten::conv2d", "aten::convolution", "aten::mm", "aten::addmm", "aten::bmm",
                                     "aten::linear", "aten::scaled_dot_product_attention") or library_kernel(n)]
    assert any("aab::flash_attn_d80_kernel" in n for n in names) and any("aab::clip_image_prep_kernel" in n for n in names)
    assert not bad, sorted(set(bad))
    assert emb.shape == (2, 1, 96) and not emb[0].any()
    assert_vs_stock(record_parity(f"SVD {which} pipeline image embedding", "image_embeds", emb[1], want, stock),
                    max_factor=2.5)
    assert isinstance(pipe._clip_image_encoder(), CLIPVisionModelWithProjection)
    assert pipe._clip_image_encoder() is pipe._clip_image_encoder()             # mirrored once
    # frames: bit-identical to the same call given our mirror's embedding
    g = torch.Generator().manual_seed(6)
    lat0 = torch.randn(1, 6, 4, 16, 24, generator=g)
    kw = dict(height=128, width=192, num_frames=6, num_inference_steps=2, decode_chunk_size=3, noise_aug_strength=0.0,
              latents=lat0, return_dict=False, output_type="pt")
    if which == "mask":
        kw["mask"] = (torch.rand(1, 16, 24, generator=g) > 0.5).float()
    else:
        m = (torch.rand(1, 6, 1, 16, 24, generator=g) > 0.5).float()
        m[:, 0] = 0
        kw["mask"] = m
    frames = pipe(pil, **kw)
    mirror_emb = pipe._clip_image_encoder().encode_images(torch.from_numpy(np.array(pil))[None].cuda(), fe.image_mean,
                                                          fe.image_std).image_embeds
    frames_e = pipe(pil, image_embeddings=mirror_emb[:, None], **kw)
    torch.cuda.synchronize()
    assert torch.equal(frames[0], frames_e[0])
