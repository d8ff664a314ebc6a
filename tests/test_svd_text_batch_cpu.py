"""CPU: `TextStableVideoDiffusionPipeline.__call__` with several images per call.  The oracle loops against the verbatim-reference
fixture `tests/golden/svd_text_batch_pipeline_tiny_ref.pt` (two videos per call; 9-channel with and without `condition_latent`,
8-channel, and a decode chunk that straddles the two videos), the mirror's host wiring over the plain-torch kernel stand-ins of
tests/ops_emulation.py against the same fixture, and the reference's errors raised before any launch."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

from ops_emulation import emulated_ops  # noqa: E402
from oracle.composition import fill_deterministic  # noqa: E402
from make_golden_svd_text_batch import CASES, call_kwargs  # noqa: E402


def _gold():
    return torch.load(os.path.join(HERE, "golden", "svd_text_batch_pipeline_tiny_ref.pt"))


def _unet_config(gold, case):
    return gold["unet_config_8ch"] if case == "stock8" else gold["unet_config"]


def _oracle_run(gold, case, decode_chunk_size=None):
    """The oracle loop of `case` from the encoded images: (frames [2, 3, F, H, W] fp32, latents [2, F, 4, h, w])."""
    from make_golden import SvdImageEncoderStub
    from oracle.composition import (AutoencoderKLTemporalDecoder, EulerDiscreteScheduler, SVD_SCHED,
                                    UNetSpatioTemporalConditionModel, oracle_svd_sampling_loop)
    from oracle.svd_stock import oracle_svd_stock_sampling_loop
    unet = fill_deterministic(UNetSpatioTemporalConditionModel(**_unet_config(gold, case)).eval(), 0)
    vae = fill_deterministic(AutoencoderKLTemporalDecoder(**gold["vae_config"]).eval(), 1)
    enc = fill_deterministic(SvdImageEncoderStub().eval(), 2)
    kw = call_kwargs(case, gold)
    noise = torch.randn(gold["image"].shape, generator=torch.Generator().manual_seed(gold["noise_seed"]))
    with torch.no_grad():
        emb = enc(gold["image"]).unsqueeze(1)                                       # [2, 1, D]
        il = vae.encode(gold["image"] + gold["noise_aug_strength"] * noise).latent_dist.mode()      # [2, 4, h, w]
    okw = dict(num_inference_steps=kw["num_inference_steps"], fps=gold["fps"] - 1, motion_bucket_id=gold["motion_bucket_id"],
               noise_aug_strength=gold["noise_aug_strength"], decode_chunk_size=decode_chunk_size or kw["decode_chunk_size"])
    if case == "stock8":
        return oracle_svd_stock_sampling_loop(unet, EulerDiscreteScheduler(**SVD_SCHED), vae, emb, il, gold["latents_in"], **okw)
    return oracle_svd_sampling_loop(unet, EulerDiscreteScheduler(**SVD_SCHED), vae, emb, il, None, gold["latents_in"],
                                    frame_mask=gold["mask"], condition_latent=kw.get("condition_latent"), **okw)


def _videos(frames):
    """oracle frames [B, 3, F, H, W] -> the reference's "pt" output [B, F, 3, H, W] in [0, 1]."""
    return (frames.permute(0, 2, 1, 3, 4) / 2 + 0.5).clamp(0, 1)


# ---------------------------------------------------------------------------------------------- oracle pin
@pytest.mark.parametrize("case", CASES)
def test_batched_text_call_oracle_matches_reference(case):
    """The oracle loops, unchanged, at batch 2: per-item images, masks and condition latents, one noise draw over the image
    batch, the CFG halves [uncond x B, cond x B], and the decode over the flattened frame axis."""
    gold = _gold()
    frames, lat = _oracle_run(gold, case)
    want = gold[f"{case}_latents"]
    assert lat.shape == want.shape == (2, 5, 4, 8, 8) and torch.isfinite(want).all()
    assert torch.allclose(lat, want, rtol=1e-5, atol=1e-5), float((lat - want).abs().max())
    if case == "straddle":
        got = _videos(frames)
        want = gold["straddle_frames"]
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-5), float((got - want).abs().max())


def test_fixture_cases_differ():
    """Each case pins something of its own: the items of a batch differ, condition_latent / image latents / 8 channels give
    other latents, and the straddling decode gives another video than the decode in whole videos."""
    gold = _gold()
    lat = {c: gold[f"{c}_latents"] for c in CASES}
    assert torch.equal(lat["condlat"], lat["straddle"])
    for a, b in (("condlat", "image"), ("condlat", "stock8"), ("image", "stock8")):
        assert float((lat[a] - lat[b]).abs().mean()) > 1e-2, (a, b)
    assert float((lat["condlat"][0] - lat["condlat"][1]).abs().mean()) > 1e-2
    whole, _ = _oracle_run(gold, "straddle", decode_chunk_size=5)
    assert float((_videos(whole) - gold["straddle_frames"]).abs().max()) > 1e-3
    assert gold["nvp2_error"][0] == "RuntimeError" and "Sizes of tensors must match" in gold["nvp2_error"][1]
    assert gold["mask_batch_error"][0] == "RuntimeError" and "Sizes of tensors must match" in gold["mask_batch_error"][1]


# ---------------------------------------------------------------------------------------------- host wiring
def _finalize_u8_standin(y, b, f, h, w, bf16, round_half_even=False):
    """ops.vae_dec_finalize_u8 stand-in for fp32 host models: the rounding the flag selects, on the fp32 values."""
    v = y[:, :3].float().reshape(b, f, h, w, 3)
    v = (v / 2 + 0.5).clamp(0, 1) * 255
    v = (v.round() if round_half_even else v).to(torch.uint8)
    return v.permute(1, 2, 0, 3, 4).reshape(f, h, b * w, 3).contiguous()


def _mirror(gold, case):
    """The stock pipeline object that app_svd.py builds; the tests call `TextStableVideoDiffusionPipeline.__call__` on it
    unbound, as app_svd.py:120 does."""
    from make_golden import SvdImageEncoderStub
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.pipeline_svd import StableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    from oracle.composition import SVD_SCHED
    unet = fill_deterministic(UNetSpatioTemporalConditionModel(**_unet_config(gold, case)).eval(), 0)
    vae = fill_deterministic(AutoencoderKLTemporalDecoder(**gold["vae_config"]).eval(), 1)
    for m in (unet, vae):
        m.__dict__["_aab_prepared"] = m._build_prepared(torch.float32, torch.device("cpu"))
    enc = fill_deterministic(SvdImageEncoderStub().eval(), 2)
    return StableVideoDiffusionPipeline(vae=vae, image_encoder=enc, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))


@pytest.mark.parametrize("case", CASES)
def test_batched_text_call_host_wiring_matches_reference(case, monkeypatch):
    from animate_anything_b200 import ops
    from animate_anything_b200.pipeline_svd import TextStableVideoDiffusionPipeline
    gold = _gold()
    rf, _ = _oracle_run(gold, case)
    want = _videos(rf)
    if case == "straddle":
        want = gold["straddle_frames"]
    kw = call_kwargs(case, gold)
    with emulated_ops():
        monkeypatch.setattr(ops, "vae_dec_finalize_u8", _finalize_u8_standin)
        stock = _mirror(gold, case)
        pipe = lambda *a, **k: TextStableVideoDiffusionPipeline.__call__(stock, *a, **k)      # noqa: E731
        out = {t: pipe(gold["image"], output_type=t, generator=torch.Generator().manual_seed(gold["noise_seed"]), **kw)
               for t in ("latent", "pt", "pil")}
    lat, rl = out["latent"], gold[f"{case}_latents"]
    assert lat.shape == rl.shape == (2, 5, 4, 8, 8)
    err = float((lat - rl).abs().max())
    assert err < 5e-4 * max(1.0, float(rl.abs().mean())), err
    assert len(out["pt"]) == len(out["pil"]) == 2
    for v in range(2):
        got = out["pt"][v]
        assert got.shape == want[v].shape == (5, 3, 64, 64)
        assert float((got - want[v]).abs().max()) < 5e-4, (v, float((got - want[v]).abs().max()))
        # "pil": the chunked uint8 path, regrouped per video, is exactly the host postprocess of the "pt" video
        pil = out["pil"][v]
        assert len(pil) == 5 and all(im.size == (64, 64) and im.mode == "RGB" for im in pil)
        ref = (got.permute(0, 2, 3, 1).numpy() * 255).round().astype(np.uint8)
        assert np.array_equal(np.stack([np.asarray(im) for im in pil]), ref)


def test_batched_text_call_rejects_before_any_launch(monkeypatch):
    """The errors the reference raises (recorded in the fixture) and the kernels' batch limit, raised before the CLIP tower,
    the VAE or any kernel runs."""
    from animate_anything_b200 import _lib, ops
    from animate_anything_b200.pipeline_svd import TextStableVideoDiffusionPipeline
    from ops_emulation import _EMULATED
    gold = _gold()
    base = call_kwargs("image", gold)
    calls = []
    with emulated_ops():
        stock = _mirror(gold, "image")
        pipe = lambda *a, **k: TextStableVideoDiffusionPipeline.__call__(stock, *a, **k)          # noqa: E731
        for k in _EMULATED:
            monkeypatch.setattr(ops, k, lambda *a, _k=k, **kw: calls.append(_k))
        monkeypatch.setattr(stock, "image_encoder", lambda *a, **k: calls.append("image_encoder"))
        n0 = _lib.launch_count()
        img = gold["image"]
        with pytest.raises(NotImplementedError, match="num_videos_per_prompt"):        # the reference: RuntimeError at :688
            pipe(img, num_videos_per_prompt=2, **base)
        with pytest.raises(RuntimeError, match="Sizes of tensors must match"):
            pipe(img, **dict(base, mask=gold["mask"][:1]))
        with pytest.raises(RuntimeError, match="Sizes of tensors must match"):
            pipe(img, **dict(base, condition_latent=gold["condition_latent"][:1]))
        with pytest.raises(RuntimeError, match="Sizes of tensors must match"):
            pipe(img, **dict(base, latents=gold["latents_in"][:1]))
        with pytest.raises(TypeError):
            pipe(img, **dict(base, mask=None))
        with pytest.raises(TypeError, match="list of generators"):
            pipe(img, generator=[torch.Generator(), torch.Generator()], **base)
        n = ops.GN_MAX_SAMPLES // 10 + 1                                               # 2 x n videos x 5 frames > 4096
        with pytest.raises(ValueError, match=f"at most {ops.GN_MAX_SAMPLES}"):
            pipe(img[:1].expand(n, -1, -1, -1), **dict(base, mask=gold["mask"][:1].expand(n, -1, -1, -1, -1), latents=None))
    assert calls == [] and _lib.launch_count() == n0
