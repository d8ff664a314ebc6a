"""A/B timing of the HBM-bound kernels at the shapes of a config-2 UNet forward (one CUDA graph of 24 calls over rotating input buffers, replay timed with events: GPU-bound like
the pipeline's graph replay; a call never finds its own input of the previous iteration in L2).  Variants are selected per PROCESS by the env
switches read in csrc (AAB_GN_TWO_PASS=1, AAB_LN_V1=1, AAB_TATTN_V1=1); run it twice to compare.
    python tools/kernel_ab.py [gn|ln|ta|fa|all]      (fa: text cross-attention)
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from animate_anything_b200 import ops  # noqa: E402

what = sys.argv[1] if len(sys.argv) > 1 else "all"
dt = torch.bfloat16
dev = "cuda"
HBM = 6485.5


def timeit(fn, nbuf, iters=24):
    """GPU-bound timing: `iters` calls captured into ONE CUDA graph (as the pipeline replays them) and the replay timed
    with events -- eager launches through ctypes are CPU-bound for kernels of a few microseconds."""
    for i in range(3):
        fn(i % nbuf)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn(0)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(iters):
            fn(i % nbuf)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (3 * iters) * 1e3      # us


tag = ",".join(k for k in ("AAB_LN_V1", "AAB_TATTN_V1") if os.environ.get(k) == "1") or "round-2 kernels"
print(f"variant: {tag}")
print("| kernel | shape | us / call | algorithmic GB/s | frac of 6485.5 |")
print("|---|---|---|---|---|")
if what in ("gn", "all"):
    for samples, rows, c in [(34, 4096, 320), (2, 69632, 320), (34, 1024, 640), (2, 17408, 640), (34, 256, 1280),
                             (2, 4352, 1280), (34, 64, 1280), (2, 1088, 1280), (34, 4096, 640)]:
        nbuf = max(2, int(300e6 // (samples * rows * c * 2)) + 1)
        nbuf = min(nbuf, 8)
        xs = [torch.randn(samples * rows, c, device=dev).to(dt) for _ in range(nbuf)]
        g = torch.ones(c, device=dev)
        b = torch.zeros(c, device=dev)
        us = timeit(lambda i: ops.groupnorm(xs[i], samples, rows, g, b, 1e-5, True), nbuf)
        by = 2.0 * 2 * samples * rows * c
        print(f"| groupnorm+silu | ({samples}, {rows}, {c}) | {us:.1f} | {by / us / 1e3:.0f} | {by / us / 1e3 / HBM:.2f} |")
        del xs
if what in ("ln", "all"):
    for rows, c in [(139264, 320), (34816, 640), (8704, 1280), (2176, 1280), (139264, 512)]:
        nbuf = min(8, max(2, int(300e6 // (rows * c * 2)) + 1))
        xs = [torch.randn(rows, c, device=dev).to(dt) for _ in range(nbuf)]
        g = torch.ones(c, device=dev)
        b = torch.zeros(c, device=dev)
        us = timeit(lambda i: ops.layernorm(xs[i], g, b), nbuf)
        by = 2.0 * 2 * rows * c
        print(f"| layernorm | ({rows}, {c}) | {us:.1f} | {by / us / 1e3:.0f} | {by / us / 1e3 / HBM:.2f} |")
        del xs
if what in ("ta", "all"):
    for b_, t, hw, heads in [(2, 17, 4096, 5), (2, 17, 1024, 10), (2, 17, 256, 20), (2, 17, 64, 20), (2, 17, 4096, 8)]:
        c = heads * 64
        rows = b_ * t * hw
        nbuf = min(8, max(2, int(300e6 // (rows * 3 * c * 2)) + 1))
        xs = [torch.randn(rows, 3 * c, device=dev).to(dt) for _ in range(nbuf)]
        us = timeit(lambda i: ops.temporal_attn_d64(xs[i], b_, t, hw, heads, 0, c, 2 * c), nbuf)
        by = 2.0 * rows * c * 4
        print(f"| temporal_attn_d64 | ({b_}, {t}, {hw}, {heads}) | {us:.1f} | {by / us / 1e3:.0f} | {by / us / 1e3 / HBM:.2f} |")
        del xs
if what in ("fa", "all"):
    for nb, heads, lq, lk in [(34, 5, 4096, 77), (34, 10, 1024, 77), (34, 20, 256, 77), (34, 20, 64, 77)]:
        c = heads * 64
        nbuf = min(8, max(2, int(300e6 // (nb * lq * c * 2)) + 1))
        qs = [torch.randn(nb * lq, c, device=dev).to(dt) for _ in range(nbuf)]
        kv = torch.randn(2 * lk, 2 * c, device=dev).to(dt)
        us = timeit(lambda i: ops.flash_attn_d64(qs[i], 0, kv, 0, c, nb, lq, lk, heads, kv_batch_div=17), nbuf)
        by = 2.0 * 2 * nb * lq * c
        fl = 4.0 * nb * heads * lq * lk * 64
        print(f"| flash cross-attn | ({nb}, {heads}, {lq}, {lk}) | {us:.1f} | {by / us / 1e3:.0f} | {by / us / 1e3 / HBM:.2f} | "
              f"{fl / us / 1e6:.0f} TFLOP/s |")
        del qs
if what in ("sa", "all"):
    # spatial self-attention of a config-2 forward (fused qkv input): L = 4096 / 1024 / 256 / 64 tokens per frame
    print("| flash self-attn | (nb, heads, L) | us / call | TFLOP/s |")
    for nb, heads, l in [(34, 5, 4096), (34, 10, 1024), (34, 20, 256), (34, 20, 64)]:
        c = heads * 64
        nbuf = 2
        qkvs = [torch.randn(nb * l, 3 * c, device=dev).to(dt) for _ in range(nbuf)]
        us = timeit(lambda i: ops.flash_attn_d64(qkvs[i], 0, qkvs[i], c, 2 * c, nb, l, l, heads), nbuf, iters=8)
        fl = 4.0 * nb * heads * l * l * 64
        print(f"| flash self-attn | ({nb}, {heads}, {l}) | {us:.1f} | {fl / us / 1e6:.0f} |")
        del qkvs
