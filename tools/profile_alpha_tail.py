"""The transparent-video tail of one config-2-sized clip (16 frames of 512x512, bf16): UNet384.decode_rgba_u8.
  python tools/profile_alpha_tail.py kernels   -> CUDA-event timing per kernel family / shape (implicit GEMM and the others)
  ncu --profile-from-start off ... python tools/profile_alpha_tail.py ncu   -> cudaProfilerStart/Stop around ONE call
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from animate_anything_b200 import ops  # noqa: E402
from animate_anything_b200.layerdiffuse_VAE import UNet384  # noqa: E402

mode = sys.argv[1] if len(sys.argv) > 1 else "kernels"
torch.manual_seed(0)
dec = UNet384().eval()
with torch.no_grad():
    for n, p in dec.named_parameters():                      # random init incl. the zero-initialised latent conv
        if p.dim() > 1:
            p.copy_(torch.randn_like(p) * (1.0 / p[0].numel()) ** 0.5)
dec = dec.to(torch.bfloat16).cuda()
g = torch.Generator().manual_seed(2)
video = torch.randn(1, 3, 16, 512, 512, generator=g).clamp(-1, 1).cuda()
latents = torch.randn(1, 4, 16, 64, 64, generator=g).bfloat16().cuda()
for _ in range(2):
    dec.decode_rgba_u8(video, latents)
torch.cuda.synchronize()
if mode == "ncu":
    torch.cuda.profiler.start()
    dec.decode_rgba_u8(video, latents)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
else:
    ops.KERNEL_PROFILE, ops.IGEMM_PROFILE = [], []
    dec.decode_rgba_u8(video, latents)
    torch.cuda.synchronize()
    kp, ip = ops.KERNEL_PROFILE, ops.IGEMM_PROFILE
    ops.KERNEL_PROFILE = ops.IGEMM_PROFILE = None
    agg = {}
    for p in kp:
        a = agg.setdefault((p["name"], str(p["shape"])), {"n": 0, "ms": 0.0, "bytes": 0.0, "flops": 0.0})
        a["n"] += 1
        a["ms"] += p["ev"][0].elapsed_time(p["ev"][1])
        a["bytes"] += p["bytes"]
        a["flops"] += p["flops"]
    for p in ip:
        key = ("igemm", f"rows={p['rows']} n={p['n']} k={p['k']} taps={p['taps']} bn={p['block_n']}")
        a = agg.setdefault(key, {"n": 0, "ms": 0.0, "bytes": 0.0, "flops": 0.0})
        a["n"] += 1
        a["ms"] += p["ev"][0].elapsed_time(p["ev"][1])
        a["bytes"] += 2.0 * p["rows"] * (p["k"] / p["taps"] + p["n"])          # one read of A + one write of D, 16-bit
        a["flops"] += p["flops"]
    print("| kernel | shape | launches | ms total | us / launch | algorithmic GB/s | TFLOP/s |")
    print("|---|---|---|---|---|---|---|")
    tot = {}
    for (name, shape), a in sorted(agg.items(), key=lambda kv: -kv[1]["ms"]):
        tot[name] = tot.get(name, 0.0) + a["ms"]
        print(f"| {name} | {shape} | {a['n']} | {a['ms']:.3f} | {1e3 * a['ms'] / a['n']:.1f} | "
              f"{a['bytes'] / a['ms'] / 1e6:.0f} | {a['flops'] / a['ms'] / 1e9:.0f} |")
    print("totals by family (ms, event-timed one by one):", {k: round(v, 3) for k, v in tot.items()})
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        dec.decode_rgba_u8(video, latents)
    e1.record()
    torch.cuda.synchronize()
    print(f"decode_rgba_u8, 16 x 512 x 512: {e0.elapsed_time(e1) / 3:.2f} ms")
