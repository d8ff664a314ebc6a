#!/usr/bin/env python3
"""One CTA per SM against two, for the short-K implicit-GEMM launches of a config-2 UNet forward.

Each configuration of each shape is timed as one CUDA graph of `--iters` launches over rotating input, residual and output
buffers (so a launch never finds the previous launch's operands in L2), replayed `--reps` times and timed with events --
per-launch eager timings of kernels this short also absorb host launch latency.  Per row: us per launch, achieved GB/s
against the HBM bound (A + B + out + residual bytes over 3.35 TB/s), and TFLOP/s.  "current" is the launch as `ops.igemm`
made it before the two-CTA rule (`ctas_per_sm=1`, the width `pick_block_n` / `fit_block_n` choose); the 64-column rows
separate the effect of the width from that of the second CTA.  The card name and power limit are read in the same call.
Needs a GPU; there is no fallback.

    python tools/igemm_short_k.py [--iters 20] [--reps 5] [--dtype bf16]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TBS = 3.35         # H100 SXM data sheet, HBM3

# (label, rows, n, k, residual, stats, geglu): the 1-tap transformer linears at the 64x64 level (2 x 17 frames x 4096 px,
# K = 320) and at the 32x32 level (K = 640)
SHAPES = [
    ("to_out/proj_out 64^2", 139264, 320, 320, True, True, False),
    ("proj_in/to_q 64^2", 139264, 320, 320, False, False, False),
    ("q|k|v 64^2", 139264, 960, 320, False, False, False),
    ("GEGLU 64^2", 139264, 2560, 320, False, False, True),
    ("to_out/proj_out 32^2", 34816, 640, 640, True, True, False),
    ("proj_in/to_q 32^2", 34816, 640, 640, False, False, False),
    ("q|k|v 32^2", 34816, 1920, 640, False, False, False),
]


def gpu_query(fields):
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=5).stdout
        return [x.strip() for x in out.strip().split(",")]
    except Exception:
        return []


def graph_time_us(torch, fn, nbuf, iters, reps):
    for i in range(nbuf):
        fn(i)
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
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / iters)
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="launches captured into one graph")
    ap.add_argument("--reps", type=int, default=5, help="graph replays; the median is reported")
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp16"])
    args = ap.parse_args()
    import torch
    from animate_anything_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("igemm_short_k.py measures on the GPU and found none")
    dt = torch.bfloat16 if args.dtype == "bf16" else torch.float16
    nbuf = 3
    print("| card | power limit W | shape | rows x n x k | config | us / launch | min - max | GB/s | of HBM bound | "
          "TFLOP/s |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    g = torch.Generator(device="cuda").manual_seed(0)
    for label, rows, n, k, res, stats, geglu in SHAPES:
        n_out = n // 2 if geglu else n
        xs = [(torch.randn(rows, k, device="cuda", generator=g)).to(dt) for _ in range(nbuf)]
        rs = [(torch.randn(rows, n_out, device="cuda", generator=g)).to(dt) for _ in range(nbuf)] if res else None
        outs = [torch.empty(rows, n_out, device="cuda", dtype=dt) for _ in range(nbuf)]
        w = (torch.randn(n, k, device="cuda", generator=g) * k ** -0.5).to(dt)
        b = torch.randn(n, device="cuda", generator=g)
        # two CTAs per SM exist at 64-column tiles only (GEGLU needs 128: its accumulators do not fit 80 registers)
        configs = [("current", None, 1)] + ([] if geglu else [("1 CTA/SM, BN 64", 64, 1), ("2 CTAs/SM, BN 64", 64, 2)])
        nbytes = 2.0 * (rows * k + n * k + rows * n_out * (2 if res else 1))
        flops = 2.0 * rows * n * k
        for name, bn, cps in configs:
            def fn(i, bn=bn, cps=cps):
                ops.linear(xs[i], w, b, out=outs[i], residual=rs[i] if res else None, stats=stats, geglu=geglu,
                           block_n=bn, ctas_per_sm=cps)
            us, lo, hi = graph_time_us(torch, fn, nbuf, args.iters, args.reps)
            card = gpu_query("name,power.limit")
            if name == "current":
                ops.IGEMM_PROFILE = []
                fn(0)
                name = f"current (1 CTA/SM, BN {ops.IGEMM_PROFILE[0]['block_n']})"
                ops.IGEMM_PROFILE = None
                torch.cuda.synchronize()
            gbs = nbytes / us / 1e3
            print(f"| {card[0] if card else torch.cuda.get_device_name(0)} | {card[1] if len(card) > 1 else 'n/a'} | "
                  f"{label} | {rows} x {n} x {k}{' + res' if res else ''}{' + stats' if stats else ''} | {name} | "
                  f"{us:.1f} | {lo:.1f} - {hi:.1f} | {gbs:.0f} | {gbs / (PEAK_TBS * 1e3):.2f} | {flops / us / 1e6:.0f} |",
                  flush=True)
        del xs, rs, outs


if __name__ == "__main__":
    main()
