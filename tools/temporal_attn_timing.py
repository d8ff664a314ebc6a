"""Times temporal attention (head dim 64) over clip lengths: the v2 kernel at T = 17, 25, 32 and the long-clip kernel at
T = 32 .. 128, at B = 2, 5 heads and HW = 4096 (UNet level 0 of a 512^2 clip) and HW = 9216 (SVD 576x1024).  CUDA events
after warm-up, median of `iters` launches; achieved TB/s counts the algorithmic bytes (q, k, v read once, out written once)
and TFLOP/s the 4 * T^2 * 64 multiply-adds per (b, pixel, head).  Then one SVD UNet forward at 78 frames with the real SVD
widths (320 / 640 / 1280, random weights, B = 2 for guidance, 64x64 latents) and the temporal attention's share of it, and
one 78-frame `TextStableVideoDiffusionPipeline` call as app_svd.py makes it (512^2, 25 steps, decode_chunk_size 7, full-size
SVD UNet and temporal VAE, random weights).  Prints the card name and power limit of the run beside the numbers.
Usage: python tools/temporal_attn_timing.py [iters] [--no-pipeline]"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from animate_anything_b200 import ops  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def kernel_table(iters):
    b, heads = 2, 5
    c = heads * 64
    print(f"{'kernel':<6}{'HW':>6}{'T':>5}{'time ms':>10}{'TB/s':>8}{'TFLOP/s':>9}")
    for hw in (4096, 9216):
        for kind, ts in (("v2", (17, 25, 32)), ("long", (32, 33, 49, 65, 78, 128))):
            fn = ops.temporal_attn_d64 if kind == "v2" else ops.temporal_attn_long
            for t in ts:
                qkv = torch.randn(b * t * hw, 3 * c, device="cuda", dtype=torch.float16)
                ms = time_ms(lambda: fn(qkv, b, t, hw, heads, 0, c, 2 * c), iters)
                nbytes = 2.0 * qkv.shape[0] * c * 4
                flops = 4.0 * b * hw * heads * t * t * 64
                print(f"{kind:<6}{hw:>6}{t:>5}{ms:>10.3f}{nbytes / ms / 1e9:>8.2f}{flops / ms / 1e9:>9.1f}")
                del qkv
    torch.cuda.empty_cache()


def svd_models(dtype):
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    torch.manual_seed(0)
    # the SVD checkpoints' widths and heads (head dim 64 everywhere), 9-channel mask UNet
    unet = UNetSpatioTemporalConditionModel(in_channels=9, num_attention_heads=(5, 10, 20, 20)).eval().to(dtype).cuda()
    vae = AutoencoderKLTemporalDecoder().eval().to(dtype).cuda()
    return unet, vae


def unet_forward(unet, iters, nf=78):
    dtype = torch.float16
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(2, nf, 9, 64, 64, device="cuda", generator=g).to(dtype)
    ehs = torch.randn(2, 1, 1024, device="cuda", generator=g).to(dtype)
    ids = torch.tensor([[6.0, 127.0, 0.02]] * 2, device="cuda")
    ms = time_ms(lambda: unet(x, 1.6378, ehs, ids), iters, warmup=2)
    ops.KERNEL_PROFILE = []
    unet(x, 1.6378, ehs, ids)
    torch.cuda.synchronize()
    rows = [r for r in ops.KERNEL_PROFILE if r["name"] == "temporal_attn_d64"]
    ops.KERNEL_PROFILE = None
    t_attn = sum(r["ev"][0].elapsed_time(r["ev"][1]) for r in rows)
    print(f"SVD UNet forward, B=2 (guidance), {nf} frames, 64x64 latents, fp16: {ms:.1f} ms (median of {iters}); temporal "
          f"attention {len(rows)} launches, {t_attn:.1f} ms = {100 * t_attn / ms:.1f} % (events around each launch)")


def pipeline_call(unet, vae, nf=78, steps=25):
    from animate_anything_b200.pipeline_svd import TextStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from oracle.composition import SVD_SCHED
    dtype = torch.float16
    g = torch.Generator().manual_seed(2)
    img = torch.randn(1, 3, 512, 512, generator=g).clamp(-1, 1)
    mask = (torch.rand(1, nf, 1, 64, 64, generator=g) > 0.5).float()
    mask[:, 0] = 0
    cl = torch.randn(1, nf, 4, 64, 64, generator=g).to(dtype)
    emb = torch.randn(1, 1, 1024, generator=g)
    pipe = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))

    def call(n):
        return TextStableVideoDiffusionPipeline.__call__(pipe, image=img, width=512, height=512, num_frames=nf,
                                                         num_inference_steps=n, decode_chunk_size=7, mask=mask,
                                                         condition_type="image", condition_latent=cl, image_embeddings=emb,
                                                         output_type="pt", return_dict=False)
    call(1)                                   # warm-up: module loads, workspaces
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    frames = call(steps)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    f = frames[0]
    print(f"TextStableVideoDiffusionPipeline.__call__, {nf} frames, 512x512, {steps} steps, decode_chunk_size 7, fp16, "
          f"random weights: {wall:.2f} s wall; frames {tuple(f.shape)}, finite {bool(torch.isfinite(f).all())}")


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    iters = int(args[0]) if args else 20
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    name, power = card()
    print(f"card: {name}, power limit {power}")
    kernel_table(iters)
    unet, vae = svd_models(torch.float16)
    unet_forward(unet, 5)
    if "--no-pipeline" not in sys.argv:
        pipeline_call(unet, vae)
    name, power = card()
    print(f"card: {name}, power limit {power} (end of run)")


if __name__ == "__main__":
    main()
