"""Kernel micro-benchmarks at the config-2 (level-0) shapes; CUDA-event timing, L2 flushed between launches.
Usage: python tools/microbench.py [names...]   (names: igemm_c320 igemm_geglu igemm_conv flash temporal gn ln)"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from animate_anything_b200 import ops  # noqa: E402

dt = torch.bfloat16
dev = "cuda"
names = sys.argv[1:] or ["igemm_c320", "igemm_c320_res", "igemm_geglu", "igemm_conv", "flash", "temporal", "gn", "ln"]
flush = torch.empty(256 * 1024 * 1024 // 4, device=dev, dtype=torch.float32)


def timeit(name, fn, bytes_=None, flops=None, iters=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    t = sorted(ts)[len(ts) // 2]
    msg = f"{name:28s} {t * 1e3:9.1f} us"
    if bytes_:
        msg += f"  {bytes_ / t / 1e6:8.1f} GB/s"
    if flops:
        msg += f"  {flops / t / 1e9:8.1f} TFLOP/s"
    print(msg, flush=True)


M = 139264
g = torch.Generator(device=dev).manual_seed(0)
rnd = lambda *s: (torch.randn(*s, device=dev, generator=g)).to(dt)
if "igemm_c320" in names or "igemm_c320_res" in names:
    x = rnd(M, 320)
    w = rnd(320, 320)
    b = torch.randn(320, device=dev)
    res = rnd(M, 320)
    if "igemm_c320" in names:
        timeit("igemm 139264x320x320", lambda: ops.linear(x, w, b), bytes_=2 * M * 320 * 2, flops=2 * M * 320 * 320)
    if "igemm_c320_res" in names:
        timeit("igemm 139264x320x320 +res", lambda: ops.linear(x, w, b, residual=res), bytes_=3 * M * 320 * 2,
               flops=2 * M * 320 * 320)
if "igemm_qkv" in names:
    x = rnd(M, 320)
    w = rnd(960, 320)
    timeit("igemm qkv 139264x960x320", lambda: ops.linear(x, w, None), bytes_=M * (320 + 960) * 2, flops=2 * M * 320 * 960)
if "igemm_geglu" in names:
    x = rnd(M, 320)
    w = rnd(2560, 320)
    b = torch.randn(2560, device=dev)
    timeit("igemm geglu 139264x2560x320", lambda: ops.linear(x, w, b, geglu=True), bytes_=M * (320 + 1280) * 2,
           flops=2 * M * 320 * 2560)
if "igemm_conv" in names:
    x = rnd(34, 64, 64, 320)
    w = rnd(320, 2880)
    b = torch.randn(320, device=dev)
    timeit("igemm conv3x3 320->320 @64x64x34", lambda: ops.conv3x3(x, w, b), flops=2 * M * 2880 * 320)
if "flash" in names:
    qkv = rnd(M, 960)
    timeit("flash self L=4096 h=5 nb=34", lambda: ops.flash_attn_d64(qkv, 0, qkv, 320, 640, 34, 4096, 4096, 5),
           flops=4 * 34 * 5 * 4096 * 4096 * 64)
    q = rnd(M, 320)
    kv = rnd(2 * 77, 640)
    timeit("flash cross Lk=77", lambda: ops.flash_attn_d64(q, 0, kv, 0, 320, 34, 4096, 77, 5, kv_batch_div=17),
           bytes_=2 * M * 320 * 2)
if "temporal" in names:
    qkv = rnd(M, 960)
    timeit("temporal attn T=17 hw=4096 h=5", lambda: ops.temporal_attn_d64(qkv, 2, 17, 4096, 5, 0, 320, 640),
           bytes_=M * (960 + 320) * 2)
if "gn" in names:
    x = rnd(M, 320)
    ga = torch.ones(320, device=dev)
    be = torch.zeros(320, device=dev)
    timeit("groupnorm 2D [34x4096,320]", lambda: ops.groupnorm(x, 34, 4096, ga, be, 1e-5, True), bytes_=3 * M * 320 * 2)
    timeit("groupnorm 3D [2x69632,320]", lambda: ops.groupnorm(x, 2, 69632, ga, be, 1e-5, True), bytes_=3 * M * 320 * 2)
if "ln" in names:
    x = rnd(M, 320)
    ga = torch.ones(320, device=dev)
    be = torch.zeros(320, device=dev)
    timeit("layernorm [139264,320]", lambda: ops.layernorm(x, ga, be), bytes_=2 * M * 320 * 2)

if "gn_shapes" in names:
    # every GroupNorm extent of config 2 (2-D per frame, 3-D per clip, concat widths, VAE decoder)
    shapes = [(32, 4096, 320), (32, 1024, 640), (32, 256, 1280), (32, 64, 1280), (32, 4096, 640), (32, 1024, 1280),
              (2, 65536, 320), (2, 16384, 640), (2, 4096, 1280), (2, 1024, 1280), (1, 65536, 320), (1, 16384, 640), (8, 262144, 128)]
    for (s_, r_, c_) in shapes:
        x = torch.randn(s_ * r_, c_, device=dev, generator=g).to(dt)
        ga = torch.ones(c_, device=dev)
        be = torch.zeros(c_, device=dev)
        timeit(f"gn [{s_}x{r_},{c_}]", lambda: ops.groupnorm(x, s_, r_, ga, be, 1e-5, True), bytes_=3 * s_ * r_ * c_ * 2)
        del x
