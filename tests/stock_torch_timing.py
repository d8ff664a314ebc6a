"""R1 baseline (BASELINE.md section 2): the SAME op sequence through stock PyTorch on the GPU — the oracle modules
(reference composition + diffusers restatement) in bf16 with cuDNN / cuBLAS / SDPA — timed with CUDA events.
This is a checker-side measurement (uses oracle/), not part of the product path."""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.composition import OracleUNet3D, AutoencoderKL, oracle_decode_latents  # noqa: E402

dev = "cuda"
dt = torch.bfloat16
torch.manual_seed(0)
with torch.device(dev):
    unet = OracleUNet3D(motion_mask=True, motion_strength=True).to(dt).eval()
    vae = AutoencoderKL().to(dt).eval()
g = torch.Generator(device=dev).manual_seed(1)
sample = torch.randn(2, 4, 16, 64, 64, device=dev, generator=g).to(dt)
cond = torch.randn(2, 4, 1, 64, 64, device=dev, generator=g).to(dt)
ehs = torch.randn(2, 77, 1024, device=dev, generator=g).to(dt)
mask = torch.ones(1, 1, 1, 64, 64, device=dev, dtype=dt)
mot = torch.tensor([4.0], device=dev)


def fwd():
    with torch.no_grad():
        return unet(sample, 500, ehs, cond, mask, motion=mot)


for _ in range(3):
    fwd()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    fwd()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 5
print(f"stock torch bf16 UNet3D forward (B=2,T=17,64x64): {ms:.2f} ms")
lat = torch.randn(1, 4, 16, 64, 64, device=dev, generator=g).to(dt)
vae.enable_slicing()
with torch.no_grad():
    oracle_decode_latents(vae, lat)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(2):
        oracle_decode_latents(vae, lat)
    e1.record()
    torch.cuda.synchronize()
vms = e0.elapsed_time(e1) / 2
print(f"stock torch bf16 VAE decode 16x512x512 (sliced): {vms:.2f} ms")
clip = 50 * ms + vms
print(f"=> stock torch clip estimate (50 steps + decode): {clip / 1e3:.2f} s = {16 / (clip / 1e3):.2f} frames/s")
