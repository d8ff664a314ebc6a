"""CPU: the stock `StableVideoDiffusionPipeline` mirror.  Checkpoint loading from the diffusers SVD layout with fp16-variant
weight files only, the stock loop's oracle against the verbatim-reference fixture, the pipeline's host wiring over the
plain-torch kernel stand-ins of tests/ops_emulation.py against that oracle, and the argument checks of the finalize
kernel's rounding flag (every call returns before a launch)."""
import ctypes as C
import json
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

SVD_UNET = dict(in_channels=8, block_out_channels=(64, 128, 128, 128), num_attention_heads=(1, 2, 2, 2),
                cross_attention_dim=64, addition_time_embed_dim=32, projection_class_embeddings_input_dim=96, num_frames=5,
                sample_size=8)
SVD_VAE = dict(block_out_channels=(64, 64, 128, 128), layers_per_block=1)   # the product VAE needs multiples of 64
CLIP = dict(hidden_size=80, intermediate_size=160, projection_dim=64, num_hidden_layers=1, num_attention_heads=1,
            image_size=28, patch_size=14)


# ---------------------------------------------------------------------------------------------- loading
def _add_variant(folder, variant="fp16"):
    """Renames every weight file of `folder` to its variant name (name.fp16.ext): the checkpoint then holds only those."""
    for n in os.listdir(folder):
        stem, ext = os.path.splitext(n)
        if ext in (".safetensors", ".bin"):
            os.rename(os.path.join(folder, n), os.path.join(folder, f"{stem}.{variant}{ext}"))


def _write_svd_checkpoint(root):
    """A tiny checkpoint in the diffusers SVD layout (model_index.json + five subfolders), fp16 weights saved under their
    variant names only.  Returns the saved state_dicts."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection as HFVision
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    from oracle.composition import SVD_SCHED
    unet = fill_deterministic(UNetSpatioTemporalConditionModel(**SVD_UNET), 0).half()
    vae = fill_deterministic(AutoencoderKLTemporalDecoder(**SVD_VAE), 1).half()
    torch.manual_seed(2)
    hf = HFVision(CLIPVisionConfig(hidden_act="gelu", **CLIP)).half()
    unet.save_pretrained(os.path.join(root, "unet"))
    vae.save_pretrained(os.path.join(root, "vae"))
    hf.save_pretrained(os.path.join(root, "image_encoder"))
    EulerDiscreteScheduler(**SVD_SCHED).save_pretrained(os.path.join(root, "scheduler"))
    os.makedirs(os.path.join(root, "feature_extractor"))
    with open(os.path.join(root, "feature_extractor", "preprocessor_config.json"), "w") as f:
        json.dump({"image_processor_type": "CLIPImageProcessor", "image_mean": [0.5, 0.4, 0.3],
                   "image_std": [0.2, 0.25, 0.3], "crop_size": {"height": 224, "width": 224}}, f)
    with open(os.path.join(root, "model_index.json"), "w") as f:
        json.dump({"_class_name": "StableVideoDiffusionPipeline", "_diffusers_version": "0.24.0",
                   "feature_extractor": ["transformers", "CLIPImageProcessor"],
                   "image_encoder": ["transformers", "CLIPVisionModelWithProjection"],
                   "scheduler": ["diffusers", "EulerDiscreteScheduler"],
                   "unet": ["diffusers", "UNetSpatioTemporalConditionModel"],
                   "vae": ["diffusers", "AutoencoderKLTemporalDecoder"]}, f)
    for sub in ("unet", "vae", "image_encoder"):
        _add_variant(os.path.join(root, sub))
    return {"unet": unet.state_dict(), "vae": vae.state_dict(),
            "image_encoder": {k: v for k, v in hf.state_dict().items() if not k.endswith("position_ids")}}


def _equal_sd(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k


def test_from_pretrained_fp16_variant(tmp_path):
    from animate_anything_b200.clip_vision import CLIPVisionModelWithProjection
    from animate_anything_b200.pipeline_svd import StableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    root = str(tmp_path)
    saved = _write_svd_checkpoint(root)
    assert not any(n.endswith((".safetensors", ".bin")) and ".fp16." not in n
                   for _, _, fs in os.walk(root) for n in fs)
    pipe = StableVideoDiffusionPipeline.from_pretrained(root, torch_dtype=torch.float16, variant="fp16")
    _equal_sd(pipe.unet.state_dict(), saved["unet"])
    _equal_sd(pipe.vae.state_dict(), saved["vae"])
    assert isinstance(pipe.image_encoder, CLIPVisionModelWithProjection)
    _equal_sd(pipe.image_encoder.state_dict(), saved["image_encoder"])
    assert isinstance(pipe.scheduler, EulerDiscreteScheduler) and pipe.scheduler.config.prediction_type == "v_prediction"
    assert pipe.feature_extractor.image_mean == [0.5, 0.4, 0.3] and pipe.feature_extractor.image_std == [0.2, 0.25, 0.3]
    assert pipe.unet.config.in_channels == 8 and pipe.vae_scale_factor == 8
    assert pipe.device == torch.device("cpu") and pipe.dtype == torch.float16
    assert pipe.to(torch.float32) is pipe and pipe.dtype == torch.float32 and pipe.vae.dtype == torch.float32


def test_from_pretrained_without_variant_names_the_missing_file(tmp_path):
    from animate_anything_b200.pipeline_svd import StableVideoDiffusionPipeline
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    root = str(tmp_path)
    _write_svd_checkpoint(root)
    with pytest.raises(FileNotFoundError, match=r"diffusion_pytorch_model\.bin"):
        StableVideoDiffusionPipeline.from_pretrained(root, torch_dtype=torch.float16)
    # a variant that is not there: both the variant files and the plain names are reported, nothing else is loaded
    with pytest.raises(FileNotFoundError, match=r"diffusion_pytorch_model\.bf16\.safetensors.*diffusion_pytorch_model\.safetensors"):
        UNetSpatioTemporalConditionModel.from_pretrained(root, subfolder="unet", variant="bf16")
    os.rename(os.path.join(root, "unet", "diffusion_pytorch_model.fp16.safetensors"),
              os.path.join(root, "unet", "diffusion_pytorch_model.safetensors"))
    with pytest.raises(FileNotFoundError, match=r"diffusion_pytorch_model\.safetensors exists"):
        UNetSpatioTemporalConditionModel.from_pretrained(root, subfolder="unet", variant="fp16")
    assert UNetSpatioTemporalConditionModel.from_pretrained(root, subfolder="unet").config.in_channels == 8


def test_from_pretrained_component_keywords_override(tmp_path):
    from animate_anything_b200.pipeline_svd import StableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    from oracle.composition import SVD_SCHED
    root = str(tmp_path)
    _write_svd_checkpoint(root)
    unet = UNetSpatioTemporalConditionModel(**dict(SVD_UNET, in_channels=9))
    sched = EulerDiscreteScheduler(**SVD_SCHED)
    fe = object()
    pipe = StableVideoDiffusionPipeline.from_pretrained(root, torch_dtype=torch.float16, variant="fp16", unet=unet,
                                                        scheduler=sched, image_encoder=None, feature_extractor=fe)
    assert pipe.unet is unet and pipe.scheduler is sched and pipe.feature_extractor is fe
    assert pipe.unet.config.in_channels == 9 and pipe.unet.dtype == torch.float32      # given components are used as-is
    assert pipe.vae.dtype == torch.float16
    # a folder-less component is None, and the other pipelines load the same way
    from animate_anything_b200.pipeline_svd import MaskStableVideoDiffusionPipeline
    import shutil
    shutil.rmtree(os.path.join(root, "image_encoder"))
    m = MaskStableVideoDiffusionPipeline.from_pretrained(root, variant="fp16")
    assert isinstance(m, MaskStableVideoDiffusionPipeline) and m.image_encoder is None and m.unet.dtype == torch.float32


# ---------------------------------------------------------------------------------------------- oracle pin
def _oracle_models(gold, vae_config=None):
    from make_golden import SvdImageEncoderStub
    from oracle.composition import AutoencoderKLTemporalDecoder, UNetSpatioTemporalConditionModel
    unet = fill_deterministic(UNetSpatioTemporalConditionModel(**gold["unet_config"]).eval(), 0)
    vae = fill_deterministic(AutoencoderKLTemporalDecoder(**(vae_config or gold["vae_config"])).eval(), 1)
    enc = fill_deterministic(SvdImageEncoderStub().eval(), 2)
    return unet, vae, enc


def _oracle_run(gold, unet, vae, enc, decode=True):
    from oracle.composition import EulerDiscreteScheduler, SVD_SCHED
    from oracle.svd_stock import oracle_svd_stock_sampling_loop
    with torch.no_grad():
        emb = enc(gold["image"]).unsqueeze(1)
        il = vae.encode(gold["image"] + gold["noise_aug_strength"] * gold["noise"]).latent_dist.mode()
    return oracle_svd_stock_sampling_loop(unet, EulerDiscreteScheduler(**SVD_SCHED), vae, emb, il, gold["latents_in"],
                                          num_inference_steps=3, fps=gold["fps"] - 1,
                                          motion_bucket_id=gold["motion_bucket_id"],
                                          noise_aug_strength=gold["noise_aug_strength"], decode_chunk_size=3, decode=decode)


def _gold():
    return torch.load(os.path.join(HERE, "golden", "svd_stock_pipeline_tiny_ref.pt"))


def test_stock_loop_matches_reference_pipeline():
    """`oracle_svd_stock_sampling_loop` vs the verbatim TextStableVideoDiffusionPipeline.__call__ with an 8-channel UNet,
    condition_type="image", no condition_latent and a NaN placeholder mask (which therefore never reached the UNet)."""
    gold = _gold()
    assert gold["unet_config"]["in_channels"] == 8
    assert torch.equal(gold["noise"], torch.randn(gold["image"].shape, generator=torch.Generator().manual_seed(gold["noise_seed"])))
    frames, lat = _oracle_run(gold, *_oracle_models(gold))
    assert torch.isfinite(gold["latents"]).all() and torch.isfinite(gold["frames"]).all()
    assert torch.allclose(lat, gold["latents"], rtol=1e-5, atol=1e-5), float((lat - gold["latents"]).abs().max())
    got = (frames[0].permute(1, 0, 2, 3) / 2 + 0.5).clamp(0, 1)
    assert torch.allclose(got, gold["frames"][0], rtol=1e-5, atol=1e-5), float((got - gold["frames"][0]).abs().max())


# ---------------------------------------------------------------------------------------------- host wiring
def _finalize_u8_standin(y, b, f, h, w, bf16, round_half_even=False):
    """ops.vae_dec_finalize_u8 stand-in for fp32 host models: the rounding the flag selects, on the fp32 values."""
    v = y[:, :3].float().reshape(b, f, h, w, 3)
    v = (v / 2 + 0.5).clamp(0, 1) * 255
    v = (v.round() if round_half_even else v).to(torch.uint8)
    return v.permute(1, 2, 0, 3, 4).reshape(f, h, b * w, 3).contiguous()


def _mirror(gold, in_channels=8):
    from make_golden import SvdImageEncoderStub
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.pipeline_svd import StableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    from oracle.composition import SVD_SCHED
    ounet, ovae, enc = _oracle_models(gold, SVD_VAE)
    unet = UNetSpatioTemporalConditionModel(**dict(gold["unet_config"], in_channels=in_channels)).eval()
    if in_channels == 8:
        unet.load_state_dict(ounet.state_dict(), strict=True)
    vae = AutoencoderKLTemporalDecoder(**SVD_VAE).eval()
    vae.load_state_dict(ovae.state_dict(), strict=True)
    for m in (unet, vae):
        m.__dict__["_aab_prepared"] = m._build_prepared(torch.float32, torch.device("cpu"))
    enc = fill_deterministic(SvdImageEncoderStub().eval(), 2)
    return StableVideoDiffusionPipeline(vae=vae, image_encoder=enc, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))


def test_stock_call_host_wiring_matches_oracle(monkeypatch):
    from animate_anything_b200 import ops
    gold = _gold()
    rf, rl = _oracle_run(gold, *_oracle_models(gold, SVD_VAE))     # the fixture's models, with a VAE the product takes
    kw = dict(height=64, width=128, num_frames=5, num_inference_steps=3, decode_chunk_size=3,
              noise_aug_strength=gold["noise_aug_strength"], fps=gold["fps"], motion_bucket_id=gold["motion_bucket_id"],
              latents=gold["latents_in"], return_dict=False)
    with emulated_ops():
        monkeypatch.setattr(ops, "vae_dec_finalize_u8", _finalize_u8_standin)
        pipe = _mirror(gold)
        out = {t: pipe(gold["image"], output_type=t, generator=torch.Generator().manual_seed(gold["noise_seed"]), **kw)
               for t in ("latent", "pt", "pil")}
    lat = out["latent"]
    assert lat.shape == rl.shape == (1, 5, 4, 8, 16)
    err = float((lat - rl).abs().max())
    assert err < 5e-4 * max(1.0, float(rl.abs().mean())), err
    want = (rf[0].permute(1, 0, 2, 3) / 2 + 0.5).clamp(0, 1)
    got = out["pt"][0]
    assert got.shape == want.shape == (5, 3, 64, 128)
    assert float((got - want).abs().max()) < 1e-3, float((got - want).abs().max())
    # "pil": the chunked uint8 path gives exactly the host postprocess of the "pt" video
    pil = out["pil"][0]
    assert len(pil) == 5 and all(im.size == (128, 64) and im.mode == "RGB" for im in pil)
    ref = (got.permute(0, 2, 3, 1).numpy() * 255).round().astype(np.uint8)
    assert np.array_equal(np.stack([np.asarray(im) for im in pil]), ref)


def test_stock_call_rejects_a_9_channel_unet_before_any_launch(monkeypatch):
    from animate_anything_b200 import _lib, ops
    from ops_emulation import _EMULATED
    gold = _gold()
    calls = []
    with emulated_ops():
        for k in _EMULATED:
            monkeypatch.setattr(ops, k, lambda *a, _k=k, **kw: calls.append(_k))
        pipe = _mirror(gold, in_channels=9)
        n0 = _lib.launch_count()
        with pytest.raises(ValueError, match="8-channel UNet"):
            pipe(gold["image"], height=64, width=128, num_frames=5, latents=gold["latents_in"])
    assert calls == [] and _lib.launch_count() == n0
    with pytest.raises(NotImplementedError, match="one video per call"):
        _mirror(gold)(torch.cat([gold["image"]] * 2), height=64, width=128, num_frames=5, image_embeddings=torch.zeros(2, 1, 64))


# ---------------------------------------------------------------------------------------------- kernel argument checks
def test_finalize_u8_rejects_unknown_flag_bits_without_a_gpu():
    from animate_anything_b200 import _lib
    lib = _lib.load()
    buf = (C.c_float * 256)()
    p = C.c_void_p(C.addressof(buf))
    for flags in (4, 5, 6, 7, 8, 11, 16, -1, -2, 1 << 30):
        assert lib.aab_vae_dec_finalize_u8(p, 8, p, 1, 1, 2, 2, flags, None) == 1, flags
