"""Wall time per video of a `TextStableVideoDiffusionPipeline` call with B = 1, 2 and 4 images, called as app_svd.py:120-133
calls it (condition_type="image", a per-frame mask and `condition_latent`, guidance), at two sizes:
  512x512, 14 frames, decode_chunk_size 7    (app_svd.py / train_svd.py)
  576x1024, 25 frames, decode_chunk_size 8   (the stock SVD-XT size; chunk size of diffusers' SVD example)
Full SVD widths (320 / 640 / 1280, heads of 64) for the 9-channel UNet and the temporal VAE, random weights, fp16.  The image
embedding is passed in (`image_embeddings`), so the CLIP tower is not timed.  Each (size, B) is warmed up with a one-step call,
then `repeats` calls are timed with a host clock around work that ends in a device synchronise; medians are printed, split
at the end of the last denoising step (a synchronise in `callback_on_step_end`) into "denoise" (image preprocessing, VAE
encode, the UNet loop) and "decode" (temporal VAE decode and the PIL frames).  The card's name, power limit and SM clock are
read with nvidia-smi at the start and at the end of the run.
Usage: python tools/svd_batch_timing.py [--steps 25] [--repeats 3] [--batches 1,2,4] [--sizes 512x512,576x1024]"""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = {"512x512": (512, 512, 14, 7), "576x1024": (576, 1024, 25, 8)}     # height, width, frames, decode_chunk_size


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def models(dtype):
    from animate_anything_b200.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    torch.manual_seed(0)
    unet = UNetSpatioTemporalConditionModel(in_channels=9, num_attention_heads=(5, 10, 20, 20)).eval().to(dtype).cuda()
    vae = AutoencoderKLTemporalDecoder().eval().to(dtype).cuda()
    return unet, vae


def time_calls(pipe, b, hh, ww, nf, chunk, steps, repeats, dtype):
    g = torch.Generator().manual_seed(b)
    img = torch.randn(b, 3, hh, ww, generator=g).clamp(-1, 1)
    mask = (torch.rand(b, nf, 1, hh // 8, ww // 8, generator=g) > 0.5).float()
    mask[:, 0] = 0                                                       # app_svd.py:111
    cl = torch.randn(b, nf, 4, hh // 8, ww // 8, generator=g).to(dtype)
    emb = torch.randn(b, 1, 1024, generator=g)
    marks = {}

    def at_step_end(p, i, t, kw):
        if i == p._num_timesteps - 1:
            torch.cuda.synchronize()
            marks["loop_end"] = time.perf_counter()
        return {}

    def call(n):
        return pipe(img, height=hh, width=ww, num_frames=nf, num_inference_steps=n, decode_chunk_size=chunk, mask=mask,
                    condition_type="image", condition_latent=cl, image_embeddings=emb,
                    generator=torch.Generator().manual_seed(7), callback_on_step_end=at_step_end, return_dict=False)

    call(1)
    torch.cuda.synchronize()
    total, denoise = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        frames = call(steps)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        total.append(t1 - t0)
        denoise.append(marks["loop_end"] - t0)
    assert len(frames) == b and all(len(v) == nf for v in frames)
    med = lambda xs: sorted(xs)[len(xs) // 2]                           # noqa: E731
    return med(total), med(denoise)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batches", default="1,2,4")
    ap.add_argument("--sizes", default=",".join(SIZES))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from animate_anything_b200.pipeline_svd import TextStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from oracle.composition import SVD_SCHED
    print(f"card (name, power limit, SM clock, max SM clock): {card()}")
    dtype = torch.float16
    unet, vae = models(dtype)
    pipe = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))
    batches = [int(b) for b in args.batches.split(",")]
    for hh, ww, nf, chunk in (SIZES[k] for k in args.sizes.split(",")):
        print(f"\n{hh}x{ww}, {nf} frames, decode_chunk_size {chunk}, {args.steps} Euler steps, fp16, median of "
              f"{args.repeats} calls after a warm-up call")
        print(f"{'B':>3}{'call s':>9}{'s/video':>9}{'denoise s/video':>17}{'decode s/video':>16}{'s/video vs B=1':>16}")
        base = None
        for b in batches:
            total, denoise = time_calls(pipe, b, hh, ww, nf, chunk, args.steps, args.repeats, dtype)
            per = total / b
            base = base or per
            print(f"{b:>3}{total:>9.2f}{per:>9.2f}{denoise / b:>17.2f}{(total - denoise) / b:>16.2f}{per / base:>16.3f}")
            torch.cuda.empty_cache()
    print(f"\ncard at the end of the run: {card()}")


if __name__ == "__main__":
    main()
