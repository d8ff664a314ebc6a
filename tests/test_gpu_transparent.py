"""GPU parity of the transparent-video branch (SURVEY row f4): `UNet384`, `LatentTransparencyOffsetEncoder`
(models/layerdiffuse_VAE.py) and `MaskedLatentToVideoPipeline.__call__` (models/pipeline_stage2.py:171-337) on the sm_90a
kernels, against (a) the outputs of the VERBATIM reference classes (tests/golden/transparent_ref.pt, fp32 math on bf16-rounded
weights), (b) the oracle restatement in fp32 on the same GPU and (c) the stock 16-bit torch execution of the same op sequence
as the yard-stick; plus the pieces that are new for this branch: the three boundary kernels (bit-exact), GroupNorm with 4
groups, and the head-dim-8 attention on the head-dim-64 flash kernel with zero-padded heads."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from util import assert_vs_stock, check, record_parity  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(HERE, "golden", "transparent_ref.pt")


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


# ---------------------------------------------------------------------------------------------- new boundary kernels
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_video_f32_to_nhwc8_and_rgba_finalize_bit_exact(dtype):
    from animate_anything_b200 import ops
    g = torch.Generator().manual_seed(0)
    video = torch.randn(2, 3, 5, 16, 24, generator=g).cuda()
    view = video[:1, :, 1:4]                                            # strided frame slice, like decode_rgba_u8 passes
    out = ops.video_f32_to_nhwc8(view, dtype)
    ref = torch.zeros(3, 16, 24, 8, dtype=dtype, device="cuda")
    ref[..., :3] = view[0].permute(1, 2, 3, 0).to(dtype)
    assert torch.equal(out, ref)
    # RGBA tail: the torch ops of models/pipeline_stage2.py:311-324 on the 16-bit decoder output
    y = (torch.randn(4 * 16 * 24, 4, generator=g) * torch.tensor([1.2, 1.2, 1.2, 0.6]) + torch.tensor([0.0, 0.0, 0.0, 0.5])).cuda()
    y[:7, 3] = torch.tensor([127.0 / 255, 127.4 / 255, 127.6 / 255, 128.0 / 255, 0.5, -1.0, 2.0], device="cuda")
    got = ops.rgba_finalize_u8(y, y.shape[0], dtype == torch.bfloat16)
    d = y.to(dtype)
    alpha = d[:, 3:] * 255.0
    alpha[alpha > 127] = 255
    alpha[alpha <= 127] = 0
    fg = (d[:, :3] + 1.0) * 127.5
    ref8 = torch.cat((fg, alpha), dim=1).float().clip(0, 255).to(torch.uint8)   # numpy clip + astype(uint8) truncation
    assert torch.equal(got, ref8), int((got != ref8).sum())


def test_pad_cols_and_cat_cols():
    from animate_anything_b200 import ops
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1000, 32, generator=g).bfloat16().cuda()
    x2 = torch.randn(1000, 64, generator=g).bfloat16().cuda()
    p = ops.pad_cols(x, 64)
    assert torch.equal(p[:, :32], x) and float(p[:, 32:].abs().max()) == 0.0
    wide = torch.randn(1000, 96, generator=g).bfloat16().cuda()
    p2 = ops.pad_cols(wide[:, :32], 64)                                   # strided source rows
    assert torch.equal(p2[:, :32], wide[:, :32]) and float(p2[:, 32:].abs().max()) == 0.0
    assert torch.equal(ops.cat_cols(x, x2), torch.cat([x, x2], dim=1))


# ---------------------------------------------------------------------------------------------- kernels at this branch's shapes
@pytest.mark.parametrize("c,rows,samples", [(32, 64 * 96, 2), (64, 32 * 48, 2), (128, 16 * 24, 3), (256, 8 * 12, 3),
                                            (96, 1024, 2), (384, 96, 2)])
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_four_groups(c, rows, samples, silu):
    from animate_anything_b200 import ops
    dtype = torch.bfloat16
    g = torch.Generator().manual_seed(c)
    x = (torch.randn(samples * rows, c, generator=g) * 1.5 + 0.3).to(dtype).cuda()
    gamma = (1 + 0.1 * torch.randn(c, generator=g)).cuda()
    beta = (0.1 * torch.randn(c, generator=g)).cuda()
    y = ops.groupnorm(x, samples, rows, gamma, beta, 1e-5, silu, 4)
    xr = x.float().view(samples, rows, c).permute(0, 2, 1)
    ref = F.group_norm(xr, 4, gamma, beta, 1e-5)
    if silu:
        ref = F.silu(ref)
    check(f"groupnorm(4) s{samples} r{rows} c{c} silu={silu}", y, ref.permute(0, 2, 1).reshape(samples * rows, c), 8e-3, 8e-4)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nb,l", [(2, 96), (3, 384), (1, 4096)])
def test_flash_zero_padded_heads_dim8(dtype, nb, l):
    """32 heads of dim 8 (UNet384's attention_head_dim) run as 32 heads of dim 64 with 56 zero columns each, scale 1/sqrt(8)."""
    from animate_anything_b200 import ops
    heads, d = 32, 8
    g = torch.Generator().manual_seed(l)
    q, k, v = (torch.randn(nb, heads, l, d, generator=g).to(dtype).cuda() for _ in range(3))
    qkv = torch.zeros(nb * l, 3 * heads * 64, dtype=dtype, device="cuda")
    for i, t in enumerate((q, k, v)):
        qkv.view(nb, l, 3, heads, 64)[:, :, i, :, :d] = t.permute(0, 2, 1, 3)
    inner = heads * 64
    out = ops.flash_attn_d64(qkv, 0, qkv, inner, 2 * inner, nb, l, l, heads, scale=d ** -0.5)
    o = out.view(nb, l, heads, 64)
    assert float(o[..., d:].abs().max()) == 0.0                           # zero V columns -> exactly zero output columns
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float())
    tol = 2e-3 if dtype == torch.float16 else 1.6e-2
    check(f"flash d8->64 nb{nb} L{l} {dtype}", o[..., :d].permute(0, 2, 1, 3), ref, tol, tol)


# ---------------------------------------------------------------------------------------------- the two models
def _load_pair(oracle_cls, ours_cls, seed, dtype):
    from oracle.composition import fill_deterministic
    oracle = fill_deterministic(oracle_cls().eval(), seed=seed)
    sd16 = {k: v.to(dtype) for k, v in oracle.state_dict().items()}
    oracle.load_state_dict({k: v.float() for k, v in sd16.items()})
    ours = ours_cls().eval()
    ours.load_state_dict(sd16, strict=True)
    return oracle.cuda(), ours.to(dtype).cuda()


def test_unet384_against_verbatim_reference_fixture():
    """bf16 sm_90a UNet384 vs the VERBATIM models/layerdiffuse_VAE.py:UNet384 output (fp32 math, same bf16-rounded weights and
    inputs), with the stock bf16 torch execution of the oracle as the yard-stick."""
    from oracle.composition import OracleUNet384
    from animate_anything_b200 import _lib
    from animate_anything_b200.layerdiffuse_VAE import UNet384
    _no_tf32()
    gold = torch.load(GOLD)
    oracle, ours = _load_pair(OracleUNet384, UNet384, 7, torch.bfloat16)
    x, lat = gold["dec_x"].cuda(), gold["dec_latent"].cuda()
    n0 = _lib.launch_count()
    y = ours(x.bfloat16(), lat.bfloat16())
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 > 150 and y.dtype == torch.bfloat16 and torch.isfinite(y).all()
    with torch.no_grad():
        ref32 = oracle(x, lat)
        stock = oracle.bfloat16()(x.bfloat16(), lat.bfloat16())
    ref = gold["dec_out"].cuda()
    assert torch.allclose(ref32, ref, rtol=1e-3, atol=1e-3)              # the oracle on this GPU reproduces the fixture
    row = record_parity("UNet384 bf16 [2,3,64,96]", "rgba (fixture)", y, ref, stock)
    assert_vs_stock(row)


@pytest.mark.parametrize("dtype,shape", [(torch.float16, (3, 128, 192)), (torch.bfloat16, (3, 128, 192)),
                                         (torch.bfloat16, (2, 512, 512))])
def test_unet384_forward(dtype, shape):
    """Whole forward against the fp32 oracle and the stock 16-bit execution; (2, 512, 512) is the production frame size:
    4096-token attention with 32 heads, 32-channel GroupNorm over 262144 pixels, producer statistics with 4 groups."""
    from oracle.composition import OracleUNet384
    from animate_anything_b200.layerdiffuse_VAE import UNet384
    _no_tf32()
    n, hh, ww = shape
    oracle, ours = _load_pair(OracleUNet384, UNet384, 7, dtype)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(n, 3, hh, ww, generator=g).clamp(-1, 1).to(dtype).cuda()
    lat = torch.randn(n, 4, hh // 8, ww // 8, generator=g).to(dtype).cuda()
    with torch.no_grad():
        ref = oracle(x.float(), lat.float())
    y = ours(x, lat)
    ours.frame_chunk = 2
    y_chunked = ours(x, lat)
    assert torch.equal(y, y_chunked)                                     # frames are independent: chunking changes nothing
    with torch.no_grad():
        stock = oracle.to(dtype)(x, lat)
    name = str(dtype).split(".")[-1]
    row = record_parity(f"UNet384 {name} [{n},3,{hh},{ww}]", "rgba", y, ref, stock)
    assert_vs_stock(row)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_offset_encoder(dtype):
    from oracle.composition import OracleLatentTransparencyOffsetEncoder
    from animate_anything_b200.layerdiffuse_VAE import LatentTransparencyOffsetEncoder
    _no_tf32()
    gold = torch.load(GOLD)
    oracle, ours = _load_pair(OracleLatentTransparencyOffsetEncoder, LatentTransparencyOffsetEncoder, 8, dtype)
    x = gold["enc_in"].cuda()
    e = ours(x.to(dtype))
    assert e.shape == (1, 4, 8, 12) and e.dtype == dtype
    with torch.no_grad():
        ref = oracle(x.to(dtype).float())
        stock = oracle.to(dtype)(x.to(dtype))
    if dtype == torch.bfloat16:
        assert torch.allclose(ref, gold["enc_out"].cuda(), rtol=1e-3, atol=1e-4)      # fixture from the verbatim class
    row = record_parity(f"OffsetEncoder {str(dtype).split('.')[-1]} [1,4,64,96]", "latent offset", e, ref, stock)
    assert_vs_stock(row)


def test_alpha_decoder_tail_timing_16x512():
    """The tail of one config-2-sized clip (16 frames of 512x512): decode_rgba_u8 timed with CUDA events; printed for DESIGN.md."""
    from oracle.composition import OracleUNet384
    from animate_anything_b200 import _lib
    from animate_anything_b200.layerdiffuse_VAE import UNet384
    _, dec = _load_pair(OracleUNet384, UNet384, 7, torch.bfloat16)
    g = torch.Generator().manual_seed(2)
    video = torch.randn(1, 3, 16, 512, 512, generator=g).clamp(-1, 1).cuda()
    latents = torch.randn(1, 4, 16, 64, 64, generator=g).bfloat16().cuda()
    out = dec.decode_rgba_u8(video, latents)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        out = dec.decode_rgba_u8(video, latents)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 3
    assert out.shape == (16, 512, 512, 4) and out.dtype == torch.uint8
    print(f"\nalpha decoder tail, 16 x 512 x 512, bf16: {ms:.2f} ms per clip, {(_lib.launch_count() - n0) // 3} kernel launches")
    from util import PARITY_ROWS
    PARITY_ROWS.append({"case": f"UNet384 tail 16x512x512 bf16: {ms:.2f} ms/clip", "stage": "timing", "ref_abs_mean": 0.0,
                        "ours_max": 0.0, "ours_mean": 0.0, "ours_viol": 0.0})


# ---------------------------------------------------------------------------------------------- the pipeline call
UNET = dict(sample_size=16, block_out_channels=(64, 128, 256, 256), attention_head_dim=64, cross_attention_dim=128,
            motion_mask=True, motion_strength=True)
VAE = dict(block_out_channels=(64, 64, 128, 128), layers_per_block=1, sample_size=128)
SCHED = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
             set_alpha_to_one=False, steps_offset=1)


def test_masked_latent_to_video_pipeline():
    """`MaskedLatentToVideoPipeline.__call__(pipeline, ...)` called UNBOUND on a base pipeline object with the keywords of
    train_transparent_i2v_stage2.py:500-515, against oracle_masked_sampling_loop (pinned on CPU to the verbatim reference call)."""
    import numpy as np
    from oracle.composition import (AutoencoderKL as OVAE, DDIMScheduler as ODDIM, OracleUNet3D, OracleUNet384,
                                    oracle_masked_sampling_loop, oracle_rgba_postprocess)
    from test_gpu_pipeline import _pair
    from animate_anything_b200 import schedulers as S
    from animate_anything_b200.autoencoder_kl import AutoencoderKL
    from animate_anything_b200.layerdiffuse_VAE import UNet384
    from animate_anything_b200.pipeline_stage2 import MaskedLatentToVideoPipeline, TextToVideoSDPipeline
    from animate_anything_b200.unet_3d_condition_mask import UNet3DConditionModel
    _no_tf32()
    dtype = torch.float16
    ounet, unet = _pair(OracleUNet3D, UNet3DConditionModel, UNET, dtype, seed=0)
    ovae, vae = _pair(OVAE, AutoencoderKL, VAE, dtype, seed=1)
    odec, dec = _load_pair(OracleUNet384, UNet384, 7, dtype)
    g = torch.Generator().manual_seed(6)
    lat = torch.randn(1, 4, 4, 16, 16, generator=g).to(dtype).cuda()
    cond = torch.randn(1, 4, 1, 16, 16, generator=g).to(dtype).cuda()
    pe = torch.randn(1, 77, 128, generator=g).to(dtype).cuda()
    ne = torch.randn(1, 77, 128, generator=g).to(dtype).cuda()
    mask1 = (torch.rand(1, 1, 1, 16, 16, generator=g) > 0.5).to(dtype).cuda()
    ref_vid, ref_lat, ref_png = oracle_masked_sampling_loop(ounet, ODDIM(**SCHED), ovae, odec, lat.float(), pe.float(),
                                                            ne.float(), cond.float(), mask1.float(), [5], 9.0, 3)
    pipeline = TextToVideoSDPipeline(vae=vae, text_encoder=None, tokenizer=None, unet=unet, scheduler=S.DDIMScheduler(**SCHED))
    video, latents, pngs, alpha_png, pngs_rgb = MaskedLatentToVideoPipeline.__call__(
        pipeline, clean_latents=lat.clone(), vae_alpha_decoder=dec, prompt_embeds=pe, negative_prompt_embeds=ne, latents=lat,
        width=128, height=128, num_frames=4, num_inference_steps=3, guidance_scale=9.0, motion=[5], return_dict=False,
        condition_latent=cond, mask=mask1)
    assert pipeline.last_gpu_launches > 1000
    assert isinstance(video, list) and len(video) == 4 and video[0].shape == (128, 128, 3) and video[0].dtype == np.uint8
    assert pngs.shape == (4, 128, 128, 4) and pngs.dtype == np.uint8
    assert (alpha_png == pngs[..., 3]).all() and (pngs_rgb == pngs[..., :3]).all() and set(np.unique(alpha_png)) <= {0, 255}
    # latents: the loop is LatentToVideoPipeline's (bounds of test_gpu_pipeline.py::test_full_loop)
    st_vid, st_lat, _ = oracle_masked_sampling_loop(ounet.to(dtype), ODDIM(**SCHED), ovae.to(dtype), odec.to(dtype), lat, pe, ne,
                                                    cond, mask1, [5], 9.0, 3)
    row = record_parity("masked pipeline fp16 4x128x128", "latents", latents, ref_lat, st_lat)
    assert_vs_stock(row, mean_factor=3.0, max_factor=4.0, mean_floor=5e-4, max_floor=5e-3)
    # the tail alone, on the pipeline's OWN latents (so that loop noise does not enter): decode + alpha decoder + RGBA bytes
    with torch.no_grad():
        from oracle.composition import oracle_decode_latents
        v32 = oracle_decode_latents(ovae.float(), latents.float())
        x = v32.permute(0, 2, 1, 3, 4).reshape(4, 3, 128, 128)
        rgba32 = odec.float()(x, latents.float().permute(0, 2, 1, 3, 4).reshape(4, 4, 16, 16))
    want = oracle_rgba_postprocess(rgba32.to(dtype), 1, 4)
    d = np.abs(pngs.astype(int) - want.astype(int))
    fg_mean, alpha_flip = float(d[..., :3].mean()), float((d[..., 3] != 0).mean())
    print(f"masked pipeline tail: foreground mean |diff| = {fg_mean:.3f} / 255, alpha pixels flipped = {alpha_flip:.4%}")
    assert fg_mean < 1.5 and alpha_flip < 0.01
    # output_type="pt" returns the fp32 video tensor (:328-329); return_dict=True the frames only (:336)
    out = MaskedLatentToVideoPipeline.__call__(pipeline, vae_alpha_decoder=dec, prompt_embeds=pe, negative_prompt_embeds=ne,
                                               latents=lat, width=128, height=128, num_frames=4, num_inference_steps=3,
                                               guidance_scale=9.0, motion=[5], condition_latent=cond, mask=mask1, output_type="pt")
    assert out.frames.shape == (1, 3, 4, 128, 128) and out.frames.dtype == torch.float32
    ev = (out.frames - ref_vid).abs()
    print(f"masked pipeline video: ref|mean|={ref_vid.abs().mean().item():.4f} max={ev.max().item():.3e} mean={ev.mean().item():.3e}")
    with pytest.raises(NotImplementedError):
        MaskedLatentToVideoPipeline.__call__(pipeline, vae_alpha_decoder=dec, prompt_embeds=pe, negative_prompt_embeds=ne,
                                             latents=lat, condition_latent=cond, mask=mask1, image_embeds=torch.zeros(1))
