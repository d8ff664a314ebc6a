"""GPU: the stock `StableVideoDiffusionPipeline` mirror and both SVD entry points of the reference run unchanged on it.

- The stock image-to-video call against `oracle.svd_stock.oracle_svd_stock_sampling_loop` (pinned to the verbatim reference on CPU by
  tests/test_svd_stock_cpu.py), fp16 and bf16, for output_type "pt", "latent" and "pil".
- The decoder tail's SVD rounding (bit 1 of `aab_vae_dec_finalize_u8`) against numpy byte for byte, and the tensor2vid
  truncation with bit 1 clear.
- Mask / Text pipelines: their "pil" frames (now rounded on the device) equal the host postprocess of their "pt" video.
- `train_svd.py --eval` (`main_eval`) and `app_svd.py` (`AnimateController`), VERBATIM excerpts written into oracle/_ref/
  by `build()` (oracle/make_ref_excerpts.py), executed on tiny fp16-variant checkpoints with the module-level names bound
  to the mirror; only imageio, gradio and accelerate's `set_seed` are stubbed.
- A profiler window over one stock call with a CLIP tower: no cuBLAS / cuDNN / SDPA kernel, only uint8 frames leave
  the device."""
import json
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from util import assert_vs_stock, record_parity  # noqa: E402

pytestmark = pytest.mark.gpu

SVD_8CH = dict(in_channels=8, block_out_channels=(64, 128, 128, 128), num_attention_heads=(1, 2, 2, 2),
               cross_attention_dim=96, addition_time_embed_dim=32, projection_class_embeddings_input_dim=96,
               num_frames=6, sample_size=16)
SVD_9CH = dict(SVD_8CH, in_channels=9)
SVD_VAE = dict(block_out_channels=(64, 64, 128, 128), layers_per_block=1)
CLIP = dict(hidden_size=80, intermediate_size=160, projection_dim=96, num_hidden_layers=1, num_attention_heads=1,
            image_size=224, patch_size=14)
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _models(dtype, unet_cfg=SVD_8CH):
    from oracle.composition import AutoencoderKLTemporalDecoder as OVAE, UNetSpatioTemporalConditionModel as OUNet
    from oracle.composition import fill_deterministic
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    ounet = fill_deterministic(OUNet(**unet_cfg).eval(), seed=0)
    ovae = fill_deterministic(OVAE(**SVD_VAE).eval(), seed=1)
    out = []
    for o, cls, cfg in ((ounet, UNetSpatioTemporalConditionModel, unet_cfg), (ovae, AutoencoderKLTemporalDecoder, SVD_VAE)):
        sd16 = {k: v.to(dtype) for k, v in o.state_dict().items()}
        o.load_state_dict({k: v.float() for k, v in sd16.items()})
        m = cls(**cfg).eval()
        m.load_state_dict(sd16, strict=True)
        out += [o.cuda(), m.to(dtype).cuda()]
    return out                                                   # ounet, unet, ovae, vae


def _host_pil(pt_frames):
    """The host tail the "pil" output used before: postprocess's numpy rounding of the [0, 1] video."""
    from animate_anything_b200.image_processor import VaeImageProcessor
    return VaeImageProcessor.numpy_to_pil(VaeImageProcessor.pt_to_numpy(pt_frames))


def _same_pil(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.mode == y.mode and x.size == y.size and x.tobytes() == y.tobytes()


# ---------------------------------------------------------------------------------------------- 1. stock call vs oracle
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_stock_call_matches_oracle(dtype):
    from oracle.composition import EulerDiscreteScheduler as OEuler, SVD_SCHED
    from oracle.svd_stock import oracle_svd_stock_sampling_loop
    from animate_anything_b200.pipeline_svd import StableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    _no_tf32()
    ounet, unet, ovae, vae = _models(dtype)
    g = torch.Generator().manual_seed(21)
    img = torch.randn(1, 3, 128, 192, generator=g).clamp(-1, 1)
    lat0 = torch.randn(1, 6, 4, 16, 24, generator=g)
    emb = torch.randn(1, 1, 96, generator=g)
    aug = 0.02
    noise = torch.randn(img.shape, generator=torch.Generator().manual_seed(22))
    pipe = StableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))
    kw = dict(height=128, width=192, num_frames=6, num_inference_steps=3, decode_chunk_size=4, noise_aug_strength=aug,
              latents=lat0, image_embeddings=emb, return_dict=False)
    out = {t: pipe(img, output_type=t, generator=torch.Generator().manual_seed(22), **kw) for t in ("pt", "latent", "pil")}
    torch.cuda.synchronize()
    assert pipe.last_gpu_launches > 300
    okw = dict(num_inference_steps=3, noise_aug_strength=aug, decode_chunk_size=4)
    with torch.no_grad():
        x_aug = (img.cuda() + aug * noise.cuda()).to(dtype)
        il32 = ovae.encode(x_aug.float()).latent_dist.mode()
        rf, rl = oracle_svd_stock_sampling_loop(ounet, OEuler(**SVD_SCHED), ovae, emb.to(dtype).float().cuda(), il32,
                                                lat0.to(dtype).float().cuda(), **okw)
        o16u, o16v = ounet.to(dtype), ovae.to(dtype)
        il16 = o16v.encode(x_aug).latent_dist.mode()
        sf, sl = oracle_svd_stock_sampling_loop(o16u, OEuler(**SVD_SCHED), o16v, emb.to(dtype).cuda(), il16,
                                                lat0.to(dtype).cuda(), **okw)
    lat = out["latent"]
    assert lat.shape == rl.shape == (1, 6, 4, 16, 24) and lat.dtype == dtype
    case = f"SVD stock pipeline {str(dtype).split('.')[-1]} 3 Euler steps"
    assert_vs_stock(record_parity(case, "latents", lat, rl, sl), mean_factor=3.0, max_factor=4.0, mean_floor=5e-4,
                    max_floor=5e-3)
    got = out["pt"][0]                                               # [F, 3, H, W] in [0, 1]
    want = (rf[0].permute(1, 0, 2, 3) / 2 + 0.5).clamp(0, 1)
    stock = (sf[0].permute(1, 0, 2, 3).float() / 2 + 0.5).clamp(0, 1)
    assert_vs_stock(record_parity(case, "frames", got, want, stock), mean_factor=3.0, max_factor=4.0, mean_floor=2e-3,
                    max_floor=2e-2)
    pil = out["pil"][0]
    assert len(pil) == 6 and all(im.size == (192, 128) and im.mode == "RGB" for im in pil)
    _same_pil(pil, _host_pil(got))                                   # device rounding == host postprocess, byte for byte
    with pytest.raises(ValueError, match="8-channel"):
        StableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=_models(dtype, SVD_9CH)[1],
                                     scheduler=EulerDiscreteScheduler(**SVD_SCHED))(img, **kw)


# ---------------------------------------------------------------------------------------------- 2. tail kernel rounding
def _all_16bit_values(dtype):
    bits = torch.arange(0, 1 << 16, dtype=torch.int32).to(torch.int16)
    v = bits.view(dtype).float()
    return v[~torch.isnan(v)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_finalize_u8_rounding_modes(dtype):
    from animate_anything_b200 import ops
    bf16 = dtype == torch.bfloat16
    g = torch.Generator().manual_seed(5)
    special = torch.tensor([0.0, -0.0, 1.0, -1.0, 1.5, -1.5, 2.0, -3.0, 1e4, -1e4, float("inf"), float("-inf")])
    # every 16-bit value (k + 0.5 ties: x = 0 gives exactly 127.5), random fp32 values that the kernel first rounds to
    # the model dtype, and values just around 0 / +-1
    vals = torch.cat([special, _all_16bit_values(dtype), torch.randn(20000, generator=g) * 1.2,
                      (torch.rand(4000, generator=g) - 0.5) * 1e-3, 1 + (torch.rand(2000, generator=g) - 0.5) * 1e-2,
                      -1 + (torch.rand(2000, generator=g) - 0.5) * 1e-2])
    b, f, h, w = 2, 3, 8, -(-vals.numel() // (3 * 2 * 3 * 8))
    n = b * f * h * w * 3
    vals = torch.cat([vals, torch.zeros(n - vals.numel())])
    y = torch.full((b * f * h * w, 8), 7.0)                           # ldc 8: columns 3.. must be ignored
    y[:, :3] = vals.view(-1, 3)
    x16 = y[:, :3].to(dtype).float().numpy()                          # what the kernel rounds to first
    half = np.clip(x16 / 2 + np.float32(0.5), 0, 1)
    want_round = (half * 255).round().astype(np.uint8)                # SVD postprocess
    want_trunc = (np.clip(x16 * np.float32(0.5) + np.float32(0.5), 0, 1) * 255).astype(np.uint8)   # tensor2vid

    def layout(a):                                                    # [b*f*h*w, 3] -> [f, h, b*w, 3]
        return a.reshape(b, f, h, w, 3).transpose(1, 2, 0, 3, 4).reshape(f, h, b * w, 3)
    yc = y.cuda()
    got_round = ops.vae_dec_finalize_u8(yc, b, f, h, w, bf16, round_half_even=True).cpu().numpy()
    got_trunc = ops.vae_dec_finalize_u8(yc, b, f, h, w, bf16).cpu().numpy()
    assert np.array_equal(got_round, layout(want_round))
    assert np.array_equal(got_trunc, layout(want_trunc))
    zero = layout(x16 == 0)[..., 0]
    assert (got_round[..., 0][zero] == 128).all() and (got_trunc[..., 0][zero] == 127).all()   # the 127.5 tie


# ---------------------------------------------------------------------------------------------- 3. Mask / Text frames
def test_mask_and_text_pil_frames_equal_host_postprocess():
    """Same inputs as tests/test_gpu_svd.py's loop tests: the "pil" frames both pipelines return now come from the
    decoder's last kernel; they equal, byte for byte, the host postprocess of the same call's "pt" video."""
    from oracle.composition import SVD_SCHED
    from animate_anything_b200.pipeline_svd import MaskStableVideoDiffusionPipeline, TextStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    _no_tf32()
    for dtype in (torch.float16, torch.bfloat16):
        _, unet, _, vae = _models(dtype, SVD_9CH)
        g = torch.Generator().manual_seed(6)
        img = torch.randn(1, 3, 128, 192, generator=g).clamp(-1, 1)
        mask = (torch.rand(1, 16, 24, generator=g) > 0.5).float()
        lat0 = torch.randn(1, 6, 4, 16, 24, generator=g)
        emb = torch.randn(1, 1, 96, generator=g)
        pipe = MaskStableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet,
                                                scheduler=EulerDiscreteScheduler(**SVD_SCHED))
        kw = dict(height=128, width=192, num_frames=6, num_inference_steps=3, decode_chunk_size=3, noise_aug_strength=0.0,
                  latents=lat0, mask=mask, image_embeddings=emb, return_dict=False)
        _same_pil(pipe(img, output_type="pil", **kw)[0], _host_pil(pipe(img, output_type="pt", **kw)[0]))
        g = torch.Generator().manual_seed(8)
        img = torch.randn(1, 3, 128, 192, generator=g).clamp(-1, 1)
        fmask = (torch.rand(1, 6, 1, 16, 24, generator=g) > 0.5).float()
        fmask[:, 0] = 0
        lat0 = torch.randn(1, 6, 4, 16, 24, generator=g)
        cl = torch.randn(1, 6, 4, 16, 24, generator=g)
        emb = torch.randn(1, 1, 96, generator=g)
        tpipe = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet,
                                                 scheduler=EulerDiscreteScheduler(**SVD_SCHED))
        kw = dict(height=128, width=192, num_frames=6, num_inference_steps=3, decode_chunk_size=3, noise_aug_strength=0.0,
                  latents=lat0, mask=fmask, image_embeddings=emb, return_dict=False, condition_type="image",
                  condition_latent=cl)
        _same_pil(tpipe(img, output_type="pil", **kw)[0], _host_pil(tpipe(img, output_type="pt", **kw)[0]))


# ---------------------------------------------------------------------------------------------- checkpoints + excerpts
class Cfg(dict):
    """attribute + item access and `.get`: what the excerpts need from the OmegaConf DictConfig."""
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


def _write_checkpoint(root, unet_cfg):
    """diffusers SVD layout with fp16-variant weight files only (a loader that ignored `variant` would fail)."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection as HFVision
    from oracle.composition import SVD_SCHED, fill_deterministic
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    fill_deterministic(UNetSpatioTemporalConditionModel(**unet_cfg), 0).half().save_pretrained(os.path.join(root, "unet"))
    fill_deterministic(AutoencoderKLTemporalDecoder(**SVD_VAE), 1).half().save_pretrained(os.path.join(root, "vae"))
    torch.manual_seed(2)
    HFVision(CLIPVisionConfig(hidden_act="gelu", **CLIP)).half().save_pretrained(os.path.join(root, "image_encoder"))
    EulerDiscreteScheduler(**SVD_SCHED).save_pretrained(os.path.join(root, "scheduler"))
    os.makedirs(os.path.join(root, "feature_extractor"))
    with open(os.path.join(root, "feature_extractor", "preprocessor_config.json"), "w") as f:
        json.dump({"image_mean": [0.48145466, 0.4578275, 0.40821073], "image_std": [0.26862954, 0.26130258, 0.27577711]}, f)
    with open(os.path.join(root, "model_index.json"), "w") as f:
        json.dump({"_class_name": "StableVideoDiffusionPipeline", "_diffusers_version": "0.24.0"}, f)
    for sub in ("unet", "vae", "image_encoder"):
        for n in os.listdir(os.path.join(root, sub)):
            stem, ext = os.path.splitext(n)
            if ext in (".safetensors", ".bin"):
                os.rename(os.path.join(root, sub, n), os.path.join(root, sub, f"{stem}.fp16{ext}"))


def _excerpt(name):
    path = os.path.join(REF_DIR, name)
    if not os.path.exists(path):
        pytest.fail(f"{path} is missing: run build() (it extracts the reference excerpts into oracle/_ref/)")
    return compile(open(path).read(), name, "exec")


def _check_clip(frames, n, w, h):
    assert len(frames) == n
    for im in frames:
        a = np.asarray(im)
        assert a.dtype == np.uint8 and a.shape == (h, w, 3)


# ---------------------------------------------------------------------------------------------- 4. train_svd.py --eval
@pytest.mark.parametrize("unet_cfg", [SVD_8CH, SVD_9CH], ids=["stock_8ch", "mask_9ch"])
def test_train_svd_main_eval_runs_unchanged(tmp_path, monkeypatch, unet_cfg):
    from typing import Dict, Optional
    import torchvision.transforms as T
    from PIL import Image
    from animate_anything_b200 import _lib
    from animate_anything_b200.pipeline_svd import MaskStableVideoDiffusionPipeline, StableVideoDiffusionPipeline
    _no_tf32()
    ckpt = str(tmp_path / "ckpt")
    _write_checkpoint(ckpt, unet_cfg)
    monkeypatch.chdir(tmp_path)                                       # main_eval writes under ./output/svd_out
    rng = np.random.default_rng(0)
    Image.fromarray((rng.random((140, 200, 3)) * 255).astype(np.uint8)).save("prompt.png")
    m = np.zeros((140, 200), dtype=np.uint8)
    m[30:110, 40:160] = 255
    Image.fromarray(m).save("prompt_label.jpg")

    written, calls = [], []
    imageio = types.SimpleNamespace(mimwrite=lambda path, frames, **kw: written.append((path, frames)))
    cls = MaskStableVideoDiffusionPipeline if unet_cfg["in_channels"] == 9 else StableVideoDiffusionPipeline
    orig = cls.__call__

    def spy(self, *a, **k):
        calls.append((self, a, k, torch.get_rng_state(), torch.cuda.get_rng_state()))
        return orig(self, *a, **k)
    monkeypatch.setattr(cls, "__call__", spy)
    ns = dict(os=os, math=math, json=json, torch=torch, np=np, T=T, Image=Image, imageio=imageio, Dict=Dict,
              Optional=Optional, set_seed=lambda s: torch.manual_seed(s),
              StableVideoDiffusionPipeline=StableVideoDiffusionPipeline,
              MaskStableVideoDiffusionPipeline=MaskStableVideoDiffusionPipeline)
    exec(_excerpt("train_svd_excerpt.py"), ns)
    vd = Cfg(prompt="", prompt_image="prompt.png", height=128, width=192, num_frames=6, num_inference_steps=3,
             decode_chunk_size=4, fps=7, motion_bucket_id=127)
    n0 = _lib.launch_count()
    ns["main_eval"](pretrained_model_path=ckpt, validation_data=vd, seed=3)
    torch.cuda.synchronize()
    assert len(calls) == 5 and len(written) == 10                     # iters = 5 clips, a .gif and a .mp4 each
    assert _lib.launch_count() - n0 > 1000, "the sm_90a kernels did not run"
    pipe = calls[0][0]
    assert type(pipe) is StableVideoDiffusionPipeline and pipe.unet.dtype == torch.float16
    assert vd.height % 64 == 0 and vd.width % 64 == 0
    for i, (self_, a, k, cpu_state, cuda_state) in enumerate(calls):
        frames = written[2 * i][1]
        assert written[2 * i + 1][1] is frames and written[2 * i][0].endswith(f"{i}.gif")
        _check_clip(frames, 6, vd.width, vd.height)
        torch.set_rng_state(cpu_state)
        torch.cuda.set_rng_state(cuda_state)
        again = orig(self_, *a, **k).frames[0]                        # a direct call from the same RNG state
        _same_pil(frames, again)
    if unet_cfg["in_channels"] == 9:
        assert tuple(calls[0][2]["mask"].shape) == (1, vd.height // 8, vd.width // 8)


# ---------------------------------------------------------------------------------------------- 5. app_svd.py
def test_app_svd_animate_controller_runs_unchanged(tmp_path, monkeypatch):
    import cv2
    import torchvision.transforms as T
    from einops import rearrange, repeat
    from PIL import Image
    from animate_anything_b200 import _lib
    from animate_anything_b200.image_processor import VaeImageProcessor
    from animate_anything_b200.pipeline_svd import StableVideoDiffusionPipeline, TextStableVideoDiffusionPipeline
    _no_tf32()
    written = []
    imageio = types.SimpleNamespace(mimwrite=lambda path, frames, **kw: written.append((path, frames, kw)))
    gr = types.SimpleNamespace(Progress=lambda *a, **k: None)
    common = dict(cv2=cv2)
    exec(_excerpt("common_excerpt.py"), common)
    ns = dict(os=os, math=math, torch=torch, Image=Image, T=T, imageio=imageio, gr=gr, rearrange=rearrange, repeat=repeat,
              VaeImageProcessor=VaeImageProcessor, StableVideoDiffusionPipeline=StableVideoDiffusionPipeline,
              TextStableVideoDiffusionPipeline=TextStableVideoDiffusionPipeline, read_video=common["read_video"])
    exec(_excerpt("app_svd_excerpt.py"), ns)
    text_calls = []
    orig_text = TextStableVideoDiffusionPipeline.__call__

    def spy(self, *a, **k):
        text_calls.append(k)
        return orig_text(self, *a, **k)
    monkeypatch.setattr(TextStableVideoDiffusionPipeline, "__call__", spy)
    rng = np.random.default_rng(1)
    bg = (rng.random((128, 128, 3)) * 255).astype(np.uint8)
    layer = np.zeros((128, 128, 4), dtype=np.uint8)
    layer[20:90, 30:100, 3] = 255
    video_path = str(tmp_path / "clip.avi")
    wr = cv2.VideoWriter(video_path, cv2.VideoWriter_fourcc(*"MJPG"), 7, (128, 128))
    for i in range(3):
        wr.write(np.roll(bg, 4 * i, axis=1)[:, :, ::-1].copy())
    wr.release()
    n0 = _lib.launch_count()
    for unet_cfg, video, nf in ((SVD_8CH, None, 6), (SVD_9CH, None, 6), (SVD_9CH, video_path, 3)):
        ckpt = str(tmp_path / f"ckpt{unet_cfg['in_channels']}")
        if not os.path.isdir(ckpt):
            _write_checkpoint(ckpt, unet_cfg)
        out_dir = str(tmp_path / "out")
        os.makedirs(out_dir, exist_ok=True)
        vd = Cfg(height=128, width=128, num_inference_steps=3, decode_chunk_size=7, fps=7, num_frames=nf,
                 motion_bucket_id=127)
        ctl = ns["AnimateController"](ckpt, vd, out_dir)
        assert type(ctl.pipeline) is StableVideoDiffusionPipeline and ctl.pipeline.unet.config.in_channels == \
            unet_cfg["in_channels"]
        n_text = len(text_calls)
        path = ctl.animate({"background": bg.copy(), "layers": [layer.copy()]}, video, 3, "5", "7", str(nf), 127)
        torch.cuda.synchronize()
        assert path == written[-1][0] and os.path.exists(os.path.join(out_dir, "0_label.jpg"))
        _check_clip(written[-1][1], nf, 128, 128)
        assert len(text_calls) == n_text + (unet_cfg["in_channels"] == 9)
        if unet_cfg["in_channels"] == 9:
            k = text_calls[-1]
            assert k["condition_type"] == "image" and tuple(k["condition_latent"].shape) == (1, nf, 4, 16, 16)
            assert tuple(k["mask"].shape) == (1, nf, 1, 16, 16) and k["decode_chunk_size"] == 7
    assert _lib.launch_count() - n0 > 1000


# ---------------------------------------------------------------------------------------------- 6. no library compute
def test_stock_call_profile_has_no_library_kernels_and_copies_only_uint8(tmp_path):
    from torch.profiler import ProfilerActivity, profile
    from PIL import Image
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection as HFVision
    from oracle.composition import SVD_SCHED
    from animate_anything_b200.clip_vision import CLIPVisionModelWithProjection
    from animate_anything_b200.pipeline_svd import StableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    _no_tf32()
    dtype = torch.float16
    _, unet, _, vae = _models(dtype)
    torch.manual_seed(2)
    enc = CLIPVisionModelWithProjection.from_hf(HFVision(CLIPVisionConfig(hidden_act="gelu", **CLIP)).eval()).to(dtype).cuda()
    pipe = StableVideoDiffusionPipeline(vae=vae, image_encoder=enc, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))
    img = Image.fromarray((np.random.default_rng(3).random((128, 192, 3)) * 255).astype(np.uint8))
    kw = dict(height=128, width=192, num_frames=6, num_inference_steps=2, decode_chunk_size=4)
    pipe(img, **kw)                                                   # weights converted outside the window
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        frames = pipe(img, **kw).frames[0]
        torch.cuda.synchronize()
    _check_clip(frames, 6, 192, 128)
    trace = str(tmp_path / "trace.json")
    prof.export_chrome_trace(trace)
    events = json.load(open(trace))["traceEvents"]
    kernels = [e["name"] for e in events if e.get("cat") == "kernel"]
    assert any("aab" in n for n in kernels)
    bad = [n for n in kernels if "aab" not in n and any(s in n.lower() for s in ("cublas", "cudnn", "gemm", "xmma", "cutlass", "flash",
                                                                   "fmha", "efficient_attention", "scaled_dot"))]
    assert not bad, sorted(set(bad))[:8]
    d2h = [int(e.get("args", {}).get("bytes", 0)) for e in events
           if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "")]
    frame_bytes = 128 * 192 * 3
    big = [x for x in d2h if x > 1024]
    assert big and max(big) <= 4 * frame_bytes and sum(big) == 6 * frame_bytes, big   # uint8 chunks of 4 + 2 frames
