"""GPU parity of the SVD leg (BASELINE config 4; SURVEY rows a23 / f3): UNetSpatioTemporalConditionModel on the sm_90a
kernels against the oracle restatement (oracle/shim/diffusers/_svd.py: leaf semantics recalled from diffusers 0.24,
PARITY UNPINNED at that level; the composition is pinned to the verbatim reference pipeline by
tests/test_oracle_golden.py::test_svd_loop_matches_reference_pipeline).  Input layout as the reference builds it at
models/pipeline.py:422: cat([mask, latents, image_latents], dim=2) -> 9 channels; CFG batch 2 with a zeroed negative
image embedding (:343)."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from util import assert_vs_stock, record_parity  # noqa: E402

pytestmark = pytest.mark.gpu

SVD_SMALL = dict(in_channels=9, block_out_channels=(64, 128, 128, 128), num_attention_heads=(1, 2, 2, 2),
                 cross_attention_dim=96, addition_time_embed_dim=32, projection_class_embeddings_input_dim=96,
                 num_frames=6, sample_size=16)
STAGES = (["conv_in"] + [f"down_blocks.{i}" for i in range(4)] + ["mid_block"] + [f"up_blocks.{i}" for i in range(4)])


def _pair(dtype):
    from oracle.composition import UNetSpatioTemporalConditionModel as OUNet, fill_deterministic
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    oracle = fill_deterministic(OUNet(**SVD_SMALL).eval(), seed=0)
    sd16 = {k: v.to(dtype) for k, v in oracle.state_dict().items()}
    oracle.load_state_dict({k: v.float() for k, v in sd16.items()})
    ours = UNetSpatioTemporalConditionModel(**SVD_SMALL).eval()
    ours.load_state_dict(sd16, strict=True)            # identical state_dict keys
    return oracle.cuda(), ours.to(dtype).cuda()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_svd_unet_forward(dtype):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _pair(dtype)
    g = torch.Generator().manual_seed(3)
    b, nf, h, w = 2, 6, 16, 24
    lat = torch.randn(1, nf, 4, h, w, generator=g)
    il = torch.randn(1, nf, 4, h, w, generator=g)
    mask = (torch.rand(1, 1, 1, h, w, generator=g) > 0.5).float().expand(2, nf, 1, h, w)
    x = torch.cat([mask, torch.cat([lat, lat]), torch.cat([torch.zeros_like(il), il])], dim=2).to(dtype).cuda()   # [2, F, 9, h, w]
    emb = torch.randn(1, 1, 96, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb]).to(dtype).cuda()
    ids = torch.tensor([[6.0, 127.0, 0.02]] * 2).cuda()
    t = torch.tensor(1.6378)
    st32, st16 = {}, {}

    def hook_into(store):
        hs = []
        for name in STAGES:
            def mk(n):
                def f(mod, args, out):
                    o = out[0] if isinstance(out, tuple) else out
                    store[n] = o.detach().float()
                return f
            hs.append(oracle.get_submodule(name).register_forward_hook(mk(name)))
        return hs
    hooks = hook_into(st32)
    with torch.no_grad():
        ref = oracle(x.float(), t, ehs.float(), ids, return_dict=False)[0]
    for hk in hooks:
        hk.remove()
    ours.__dict__["_trace"] = []
    out = ours(x, t, ehs, ids).sample
    torch.cuda.synchronize()
    trace = ours.__dict__["_trace"]
    ours.__dict__["_trace"] = None
    hooks = hook_into(st16)
    with torch.no_grad():
        stock = oracle.to(dtype)(x, t, ehs, ids.to(dtype), return_dict=False)[0].float()
    for hk in hooks:
        hk.remove()
    assert out.shape == ref.shape == (b, nf, 4, h, w) and torch.isfinite(out).all()
    case = f"SVD UNet small {str(dtype).split('.')[-1]} [2,6,9,16,24]"
    for name, xx, gg in trace:
        got = xx.float().reshape(gg.n, gg.h, gg.w, -1).permute(0, 3, 1, 2)
        row = record_parity(case, name, got, st32[name], st16[name])
        assert_vs_stock(row, mean_factor=2.0, max_factor=3.0, mean_floor=1e-3, max_floor=1e-2)
    assert_vs_stock(record_parity(case, "output", out, ref, stock))


def test_svd_unet_rejects_bad_inputs():
    _, ours = _pair(torch.float16)
    x = torch.zeros(1, 6, 9, 16, 24, dtype=torch.float16, device="cuda")
    e = torch.zeros(1, 1, 96, dtype=torch.float16, device="cuda")
    with pytest.raises(ValueError):
        ours(x, 1.0, e, torch.zeros(1, 2, device="cuda"))              # added_time_ids of the wrong length
    with pytest.raises(ValueError):
        ours(x[:, :, :8], 1.0, e, torch.zeros(1, 3, device="cuda"))     # 8 instead of 9 input channels
    with pytest.raises(ValueError):
        ours(x[..., :20], 1.0, e, torch.zeros(1, 3, device="cuda"))     # width 20: not a multiple of 8


SVD_VAE = dict(block_out_channels=(64, 64, 128, 128), layers_per_block=1)


def _vae_pair(dtype):
    from oracle.composition import AutoencoderKLTemporalDecoder as OVAE, fill_deterministic
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    ovae = fill_deterministic(OVAE(**SVD_VAE).eval(), seed=1)
    sd16 = {k: v.to(dtype) for k, v in ovae.state_dict().items()}
    ovae.load_state_dict({k: v.float() for k, v in sd16.items()})
    vae = AutoencoderKLTemporalDecoder(**SVD_VAE).eval()
    vae.load_state_dict(sd16, strict=True)
    return ovae.cuda(), vae.to(dtype).cuda()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_svd_temporal_vae(dtype):
    """AutoencoderKLTemporalDecoder: encode (mode) and chunked temporal decode against the oracle restatement."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ovae, vae = _vae_pair(dtype)
    g = torch.Generator().manual_seed(4)
    img = torch.randn(1, 3, 64, 96, generator=g).clamp(-1, 1).to(dtype).cuda()
    z = torch.randn(5, 4, 8, 12, generator=g).to(dtype).cuda()
    with torch.no_grad():
        r_enc = ovae.encode(img.float()).latent_dist.mode()
        r_dec = ovae.decode(z.float(), num_frames=5).sample
        o16 = ovae.to(dtype)
        s_enc = o16.encode(img).latent_dist.mode().float()
        s_dec = o16.decode(z, num_frames=5).sample.float()
    enc = vae.encode(img).latent_dist.mode()
    dec = vae.decode(z, num_frames=5).sample
    vid = vae.decode_chunk_video(z, 5)
    assert dec.shape == r_dec.shape == (5, 3, 64, 96) and dec.dtype == dtype
    assert torch.equal(vid[0].permute(1, 0, 2, 3).to(dtype), dec)
    case = f"SVD temporal VAE {str(dtype).split('.')[-1]}"
    assert_vs_stock(record_parity(case, "encode", enc, r_enc, s_enc), max_factor=2.5)
    assert_vs_stock(record_parity(case, "decode 5 frames", dec, r_dec, s_dec), max_factor=2.5)


def test_svd_pipeline_loop_matches_oracle():
    """MaskStableVideoDiffusionPipeline.__call__ mirror (fused input assembly, UNet, fused per-frame CFG + Euler step,
    chunked temporal decode) against `oracle_svd_sampling_loop` (pinned to the verbatim reference pipeline on CPU)."""
    from oracle.composition import EulerDiscreteScheduler as OEuler, SVD_SCHED, oracle_svd_sampling_loop
    from animate_anything_b200.pipeline_svd import MaskStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dtype = torch.float16
    ounet, unet = _pair(dtype)
    ovae, vae = _vae_pair(dtype)
    g = torch.Generator().manual_seed(6)
    img = torch.randn(1, 3, 128, 192, generator=g).clamp(-1, 1)
    mask = (torch.rand(1, 16, 24, generator=g) > 0.5).float()
    lat0 = torch.randn(1, 6, 4, 16, 24, generator=g)
    emb = torch.randn(1, 1, 96, generator=g)
    pipe = MaskStableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))
    kw = dict(height=128, width=192, num_frames=6, num_inference_steps=3, decode_chunk_size=3, noise_aug_strength=0.0,
              latents=lat0, mask=mask, image_embeddings=emb, return_dict=False)
    frames = pipe(img, output_type="pt", **kw)
    lat = pipe(img, output_type="latent", **kw)
    torch.cuda.synchronize()
    assert pipe.last_gpu_launches > 500
    with torch.no_grad():
        il32 = ovae.encode(img.to(dtype).float().cuda()).latent_dist.mode()
        rf, rl = oracle_svd_sampling_loop(ounet, OEuler(**SVD_SCHED), ovae, emb.to(dtype).float().cuda(), il32, mask.cuda(),
                                          lat0.to(dtype).float().cuda(), num_inference_steps=3, noise_aug_strength=0.0,
                                          decode_chunk_size=3)
        o16u, o16v = ounet.to(dtype), ovae.to(dtype)
        il16 = o16v.encode(img.to(dtype).cuda()).latent_dist.mode()
        sf, sl = oracle_svd_sampling_loop(o16u, OEuler(**SVD_SCHED), o16v, emb.to(dtype).cuda(), il16, mask.to(dtype).cuda(),
                                          lat0.to(dtype).cuda(), num_inference_steps=3, noise_aug_strength=0.0,
                                          decode_chunk_size=3)
    assert lat.shape == rl.shape == (1, 6, 4, 16, 24)
    case = "SVD pipeline fp16 3 Euler steps"
    assert_vs_stock(record_parity(case, "latents", lat, rl, sl), mean_factor=3.0, max_factor=4.0, mean_floor=5e-4,
                    max_floor=5e-3)
    got = frames[0]                                         # [F, 3, H, W] in [0, 1]
    want = (rf[0].permute(1, 0, 2, 3) / 2 + 0.5).clamp(0, 1)
    stock = (sf[0].permute(1, 0, 2, 3) / 2 + 0.5).clamp(0, 1)
    assert_vs_stock(record_parity(case, "frames", got, want, stock), mean_factor=3.0, max_factor=4.0, mean_floor=2e-3,
                    max_floor=2e-2)


def test_svd_text_pipeline_image_branch():
    """`TextStableVideoDiffusionPipeline.__call__` mirror, called as app_svd.py:120-133 calls the reference's (condition_type="image",
    caller-supplied per-frame `condition_latent`, per-frame mask with frame 0 cleared), and with the image's own latents: against
    the oracle loop (pinned to the verbatim reference class by tests/golden/svd_text_pipeline_tiny_ref.pt on CPU).  A multi-token
    context fails in the UNet exactly as it does under the pinned diffusers 0.24."""
    from oracle.composition import EulerDiscreteScheduler as OEuler, SVD_SCHED, oracle_svd_sampling_loop
    from animate_anything_b200.pipeline_svd import TextStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dtype = torch.float16
    ounet, unet = _pair(dtype)
    ovae, vae = _vae_pair(dtype)
    g = torch.Generator().manual_seed(8)
    img = torch.randn(1, 3, 128, 192, generator=g).clamp(-1, 1)
    mask = (torch.rand(1, 6, 1, 16, 24, generator=g) > 0.5).float()
    mask[:, 0] = 0
    lat0 = torch.randn(1, 6, 4, 16, 24, generator=g)
    cl = torch.randn(1, 6, 4, 16, 24, generator=g)
    emb = torch.randn(1, 1, 96, generator=g)
    pipe = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))
    kw = dict(height=128, width=192, num_frames=6, num_inference_steps=3, decode_chunk_size=3, noise_aug_strength=0.0,
              latents=lat0, mask=mask, image_embeddings=emb, return_dict=False, output_type="latent")
    lat_c = pipe(img, condition_type="image", condition_latent=cl, **kw)
    lat_i = pipe(img, condition_type="image", **kw)
    torch.cuda.synchronize()
    assert pipe.last_gpu_launches > 500
    okw = dict(num_inference_steps=3, noise_aug_strength=0.0, decode=False)
    with torch.no_grad():
        il32 = ovae.encode(img.to(dtype).float().cuda()).latent_dist.mode()
        m32, l32, c32 = mask.cuda(), lat0.to(dtype).float().cuda(), cl.to(dtype).float().cuda()
        e32 = emb.to(dtype).float().cuda()
        _, r_c = oracle_svd_sampling_loop(ounet, OEuler(**SVD_SCHED), ovae, e32, il32, None, l32, frame_mask=m32,
                                          condition_latent=c32, **okw)
        _, r_i = oracle_svd_sampling_loop(ounet, OEuler(**SVD_SCHED), ovae, e32, il32, None, l32, frame_mask=m32, **okw)
        o16u, o16v = ounet.to(dtype), ovae.to(dtype)
        il16 = o16v.encode(img.to(dtype).cuda()).latent_dist.mode()
        _, s_c = oracle_svd_sampling_loop(o16u, OEuler(**SVD_SCHED), o16v, emb.to(dtype).cuda(), il16, None, lat0.to(dtype).cuda(),
                                          frame_mask=mask.to(dtype).cuda(), condition_latent=cl.to(dtype).cuda(), **okw)
        _, s_i = oracle_svd_sampling_loop(o16u, OEuler(**SVD_SCHED), o16v, emb.to(dtype).cuda(), il16, None, lat0.to(dtype).cuda(),
                                          frame_mask=mask.to(dtype).cuda(), **okw)
    case = "SVD Text pipeline (image branch) fp16 3 Euler steps"
    assert_vs_stock(record_parity(case, "latents, condition_latent", lat_c, r_c, s_c), mean_factor=3.0, max_factor=4.0,
                    mean_floor=5e-4, max_floor=5e-3)
    assert_vs_stock(record_parity(case, "latents, image latents", lat_i, r_i, s_i), mean_factor=3.0, max_factor=4.0,
                    mean_floor=5e-4, max_floor=5e-3)
    # the two branches really differ (condition_latent feeds both CFG halves, the image latents only the conditional one)
    assert (lat_c.float() - lat_i.float()).abs().mean().item() > 1e-2
    with pytest.raises(RuntimeError, match="expanded size of the tensor"):
        pipe(img, condition_type="text", prompt_embeds=torch.randn(1, 7, 96), negative_prompt_embeds=torch.randn(1, 7, 96),
             **{k: v for k, v in kw.items() if k != "image_embeddings"})
    with pytest.raises(TypeError):
        pipe(img, condition_type="image", **{**kw, "mask": None})


def test_svd_in_assemble_frames_kernel():
    """`aab_svd_in_assemble_frames` against the torch statement of models/pipeline.py:590,596-606,654-661 (per-frame mask and
    conditioning latents, zero or duplicated unconditional half, 9- and 8-channel inputs)."""
    from animate_anything_b200 import ops
    g = torch.Generator().manual_seed(1)
    for dtype in (torch.float16, torch.bfloat16):
        x = torch.randn(1, 5, 4, 8, 12, generator=g).to(dtype).cuda()
        cond_f = torch.randn(1, 1, 5, 4, 8, 12, generator=g).to(dtype).cuda()
        cond_1 = torch.randn(1, 1, 1, 4, 8, 12, generator=g).to(dtype).cuda()
        mask = (torch.rand(1, 5, 8, 12, generator=g) > 0.5).to(dtype).cuda()
        sigma = 3.7
        xs = (x.float() * torch.tensor(1.0 / (sigma * sigma + 1.0) ** 0.5, dtype=torch.float32)).to(dtype)   # the kernel's form
        for cond, zero_uncond, m in ((cond_f, False, mask), (cond_1, True, mask), (cond_f, False, None), (cond_1, True, None)):
            for cfg in (True, False):
                out = ops.svd_in_assemble_frames(x, cond, m, sigma, cfg, zero_uncond)
                c5 = cond[0].expand(1, 5, 4, 8, 12)
                if cfg:
                    cc = torch.cat([torch.zeros_like(c5) if zero_uncond else c5, c5])
                    xx = torch.cat([xs, xs])
                    mm = None if m is None else torch.cat([m, m])[:, :, None]
                else:
                    cc, xx, mm = c5, xs, None if m is None else m[:, :, None]
                want = torch.cat(([mm] if mm is not None else []) + [xx, cc], dim=2)           # [B', F, 9|8, h, w]
                nch = want.shape[2]
                got = out.view(want.shape[0], 5, 8, 12, 16).permute(0, 1, 4, 2, 3)
                assert torch.equal(got[:, :, :nch], want), (dtype, zero_uncond, m is None, cfg)
                assert not got[:, :, nch:].any()
