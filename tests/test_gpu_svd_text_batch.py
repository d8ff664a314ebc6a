"""GPU: `TextStableVideoDiffusionPipeline.__call__` with several images per call on the sm_90a kernels.
- The four two-video cases of tests/golden/svd_text_batch_pipeline_tiny_ref.pt (pinned to the verbatim reference class on CPU by
  tests/test_svd_text_batch_cpu.py) against the oracle loops, in fp16 and bf16.
- The SVD UNet at batch 4 and 8, where the temporal cross-attention's context index (b * S + s) % B depends on the batch.
- The GEGLU linear of the top-level transformers at the row count of a four-video call at 576x1024 x 25 frames (a 1,280-wide
  output of 2.36e9 elements, more than 2^31) and the linear that reads it, against a chunked torch reference.
- A two-step four-video call at 576x1024 x 25 frames with the SVD widths returns finite frames."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
from util import assert_vs_stock, record_parity  # noqa: E402
from make_golden_svd_text_batch import CASES, call_kwargs  # noqa: E402

pytestmark = pytest.mark.gpu


def _gold():
    return torch.load(os.path.join(HERE, "golden", "svd_text_batch_pipeline_tiny_ref.pt"))


def _models(gold, case, dtype):
    """(oracle UNet, oracle VAE) in fp32 holding `dtype`-rounded weights, and the product pair with the same weights."""
    from oracle.composition import (AutoencoderKLTemporalDecoder as OVAE, UNetSpatioTemporalConditionModel as OUNet,
                                    fill_deterministic)
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    ucfg = gold["unet_config_8ch"] if case == "stock8" else gold["unet_config"]
    pairs = []
    for ocls, cls, cfg, seed in ((OUNet, UNetSpatioTemporalConditionModel, ucfg, 0),
                                 (OVAE, AutoencoderKLTemporalDecoder, gold["vae_config"], 1)):
        o = fill_deterministic(ocls(**cfg).eval(), seed)
        sd16 = {k: v.to(dtype) for k, v in o.state_dict().items()}
        o.load_state_dict({k: v.float() for k, v in sd16.items()})
        m = cls(**cfg).eval()
        m.load_state_dict(sd16, strict=True)
        pairs.append((o.cuda(), m.to(dtype).cuda()))
    return pairs


def _oracle(gold, case, unet, vae, enc, dtype, compute):
    """The oracle loop of `case` with the product's roundings of the inputs; `compute` = torch.float32 (reference) or
    `dtype` (the stock 16-bit execution)."""
    from oracle.composition import EulerDiscreteScheduler, SVD_SCHED, oracle_svd_sampling_loop
    from oracle.svd_stock import oracle_svd_stock_sampling_loop
    kw = call_kwargs(case, gold)
    noise = torch.randn(gold["image"].shape, generator=torch.Generator().manual_seed(gold["noise_seed"]))
    r = lambda t: t.to(dtype).to(compute).cuda()                               # noqa: E731
    with torch.no_grad():
        emb = r(enc(gold["image"].cuda()).unsqueeze(1))
        il = vae.encode(r(gold["image"] + gold["noise_aug_strength"] * noise)).latent_dist.mode()
        okw = dict(num_inference_steps=kw["num_inference_steps"], fps=gold["fps"] - 1,
                   motion_bucket_id=gold["motion_bucket_id"], noise_aug_strength=gold["noise_aug_strength"],
                   decode_chunk_size=kw["decode_chunk_size"])
        if case == "stock8":
            return oracle_svd_stock_sampling_loop(unet, EulerDiscreteScheduler(**SVD_SCHED), vae, emb, il,
                                                  r(gold["latents_in"]), **okw)
        cl = kw.get("condition_latent")
        return oracle_svd_sampling_loop(unet, EulerDiscreteScheduler(**SVD_SCHED), vae, emb, il, None, r(gold["latents_in"]),
                                        frame_mask=r(gold["mask"]), condition_latent=None if cl is None else r(cl), **okw)


def _videos(frames):
    return (frames.permute(0, 2, 1, 3, 4) / 2 + 0.5).clamp(0, 1)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_batched_text_call_matches_oracle(dtype, case):
    from make_golden import SvdImageEncoderStub
    from oracle.composition import fill_deterministic
    from animate_anything_b200.pipeline_svd import TextStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from oracle.composition import SVD_SCHED
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    gold = _gold()
    (ounet, unet), (ovae, vae) = _models(gold, case, dtype)
    enc = fill_deterministic(SvdImageEncoderStub().eval(), 2).cuda()
    pipe = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=enc, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))
    kw = call_kwargs(case, gold)
    gen = lambda: torch.Generator().manual_seed(gold["noise_seed"])          # noqa: E731
    lat = pipe(gold["image"], output_type="latent", generator=gen(), **kw)
    frames = pipe(gold["image"], output_type="pt", generator=gen(), **kw)
    torch.cuda.synchronize()
    rf, rl = _oracle(gold, case, ounet, ovae, enc, dtype, torch.float32)
    sf, sl = _oracle(gold, case, ounet.to(dtype), ovae.to(dtype), enc, dtype, dtype)
    assert lat.shape == rl.shape == (2, 5, 4, 8, 8) and len(frames) == 2
    name = f"SVD Text pipeline, 2 videos, {case}, {str(dtype).split('.')[-1]}, 3 Euler steps"
    assert_vs_stock(record_parity(name, "latents", lat, rl, sl), mean_factor=3.0, max_factor=4.0, mean_floor=5e-4,
                    max_floor=5e-3)
    got = torch.stack([f.cuda() for f in frames])
    assert_vs_stock(record_parity(name, "frames", got, _videos(rf), _videos(sf.float())), mean_factor=3.0, max_factor=4.0,
                    mean_floor=2e-3, max_floor=2e-2)


SVD_SMALL = dict(in_channels=9, block_out_channels=(64, 128, 128, 128), num_attention_heads=(1, 2, 2, 2),
                 cross_attention_dim=96, addition_time_embed_dim=32, projection_class_embeddings_input_dim=96,
                 num_frames=6, sample_size=16)


@pytest.mark.parametrize("batch", [4, 8])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_svd_unet_forward_large_batch(dtype, batch):
    """UNet batch 4 / 8 (two / four videos under guidance), a different image embedding per video: the temporal blocks'
    cross-attention reads the context of sample (b * S + s) % B, which mixes the videos' embeddings differently at every
    batch size."""
    from oracle.composition import UNetSpatioTemporalConditionModel as OUNet, fill_deterministic
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle = fill_deterministic(OUNet(**SVD_SMALL).eval(), seed=0)
    sd16 = {k: v.to(dtype) for k, v in oracle.state_dict().items()}
    oracle.load_state_dict({k: v.float() for k, v in sd16.items()})
    ours = UNetSpatioTemporalConditionModel(**SVD_SMALL).eval()
    ours.load_state_dict(sd16, strict=True)
    oracle, ours = oracle.cuda(), ours.to(dtype).cuda()
    g = torch.Generator().manual_seed(9)
    nf, h, w = 6, 16, 24
    x = torch.randn(batch, nf, 9, h, w, generator=g)
    x[:, :, :1] = (x[:, :, :1] > 0).float()                                  # mask channel
    emb = torch.randn(batch // 2, 1, 96, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb]).to(dtype).cuda()
    ids = torch.tensor([[6.0, 127.0, 0.02]] * batch).cuda()
    x = x.to(dtype).cuda()
    t = torch.tensor(1.6378)
    with torch.no_grad():
        ref = oracle(x.float(), t, ehs.float(), ids, return_dict=False)[0]
    out = ours(x, t, ehs, ids).sample
    torch.cuda.synchronize()
    with torch.no_grad():
        stock = oracle.to(dtype)(x, t, ehs, ids.to(dtype), return_dict=False)[0].float()
    assert out.shape == ref.shape == (batch, nf, 4, h, w) and torch.isfinite(out).all()
    assert_vs_stock(record_parity(f"SVD UNet small {str(dtype).split('.')[-1]} batch {batch}", "output", out, ref, stock))


def test_geglu_linear_above_2_31_elements():
    """The top-level GEGLU feed-forward of a four-video call at 576x1024 x 25 frames: 2 x 4 x 25 x 72 x 128 = 1,843,200 rows,
    320 -> 2 x 1,280 (values | gates) -> 1,280 (2.36e9 output elements), then the 1,280 -> 320 linear with the residual that
    reads it.  Rows past element 2^31 are compared like the first ones, against torch in fp32, 65,536 rows at a time."""
    from animate_anything_b200 import ops
    torch.backends.cuda.matmul.allow_tf32 = False
    dtype = torch.float16
    m, k, n = 1_843_200, 320, 2560
    assert m * n // 2 > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(m, k, device="cuda", generator=g).to(dtype)
    w1 = (torch.randn(n, k, device="cuda", generator=g) * k ** -0.5).to(dtype)
    b1 = torch.randn(n, device="cuda", generator=g) * 0.5
    w2 = (torch.randn(k, n // 2, device="cuda", generator=g) * (n // 2) ** -0.5).to(dtype)
    b2 = torch.randn(k, device="cuda", generator=g) * 0.5
    res = torch.randn(m, k, device="cuda", generator=g).to(dtype)
    f = ops.linear(x, w1, b1, geglu=True)
    y = ops.linear(f, w2, b2, residual=res)
    torch.cuda.synchronize()
    assert f.shape == (m, n // 2) and y.shape == (m, k)
    worst_f = worst_y = 0.0
    step = 65536
    for r0 in range(0, m, step):
        full = x[r0: r0 + step].float() @ w1.float().t() + b1
        ref_f = full[:, : n // 2] * F.gelu(full[:, n // 2:])
        got_f = f[r0: r0 + step].float()
        worst_f = max(worst_f, float(((got_f - ref_f).abs() / (1e-3 + 4e-3 * ref_f.abs())).max()))
        ref_y = got_f @ w2.float().t() + b2 + res[r0: r0 + step].float()   # the second linear on the first one's output
        got_y = y[r0: r0 + step].float()
        worst_y = max(worst_y, float(((got_y - ref_y).abs() / (1e-3 + 4e-3 * ref_y.abs())).max()))
    assert worst_f <= 1.0, worst_f
    assert worst_y <= 1.0, worst_y


def test_four_videos_at_576x1024_25_frames_are_finite():
    """A two-step `TextStableVideoDiffusionPipeline` call with four images at the stock SVD size (UNet batch 8 = 200 frames,
    1,843,200 rows at the top level), the SVD widths with random weights, fp16, decode in chunks of 8 frames."""
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.pipeline_svd import TextStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    from oracle.composition import SVD_SCHED
    dtype, b, nf, hh, ww = torch.float16, 4, 25, 576, 1024
    torch.manual_seed(0)
    unet = UNetSpatioTemporalConditionModel(in_channels=9, num_attention_heads=(5, 10, 20, 20)).eval().to(dtype).cuda()
    vae = AutoencoderKLTemporalDecoder().eval().to(dtype).cuda()
    pipe = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))
    g = torch.Generator().manual_seed(4)
    img = torch.randn(b, 3, hh, ww, generator=g).clamp(-1, 1)
    mask = (torch.rand(b, nf, 1, hh // 8, ww // 8, generator=g) > 0.5).float()
    mask[:, 0] = 0
    emb = torch.randn(b, 1, 1024, generator=g)
    frames = pipe(img, height=hh, width=ww, num_frames=nf, num_inference_steps=2, decode_chunk_size=8, mask=mask,
                  image_embeddings=emb, generator=torch.Generator().manual_seed(5), output_type="pt", return_dict=False)
    torch.cuda.synchronize()
    assert len(frames) == b
    for v in frames:
        assert v.shape == (nf, 3, hh, ww) and bool(torch.isfinite(v).all())
