#!/usr/bin/env python3
"""Where the implicit-GEMM time of one config-2 UNet forward goes, one row per distinct launch shape.

Builds the UNet exactly as bench.py does, runs one eager forward with every implicit-GEMM launch bracketed by CUDA events
and prints, per (rows, n, k, taps, tile width, epilogue flavour): launches, time, share, TFLOP/s on useful flops, the tile
grid and its waves, useful / issued columns, and a lower bound from the shapes alone -- the larger of issued flops over the
data-sheet 989 TFLOP/s and (A + B + out + residual) bytes over 3.35 TB/s.  Needs a GPU; there is no fallback.

    python tools/igemm_shapes.py [--reps 3]
"""
import argparse
import collections
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS = 989.0     # H100 SXM data sheet, dense bf16 / fp16
PEAK_TBS = 3.35         # H100 SXM data sheet, HBM3


def gpu_query(fields):
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=5).stdout
        return [x.strip() for x in out.strip().split(",")]
    except Exception:
        return []


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="profiled forwards; the per-launch median is reported")
    args = ap.parse_args()
    import torch
    import bench
    from animate_anything_b200 import _lib, ops
    if not torch.cuda.is_available():
        raise SystemExit("igemm_shapes.py measures on the GPU and found none")
    dev = torch.device("cuda", 0)
    pipe = bench.build_models(dev, torch.bfloat16)
    devin = {k: v.to(dev) for k, v in bench.synth_inputs(0, pinned=False).items()}
    sample = devin["latents"].expand(2, -1, -1, -1, -1)
    cond2 = torch.cat([devin["condition_latent"]] * 2)
    ehs = torch.cat([devin["negative_prompt_embeds"], devin["prompt_embeds"]])
    tt = torch.tensor([500.0], device=dev)
    mot = torch.tensor([4.0], device=dev)

    def fwd():
        pipe.unet(sample, tt, ehs, condition_latent=cond2, mask=devin["mask"], motion=mot, _raw_eps=True)

    with torch.no_grad():
        for _ in range(2):
            fwd()
        torch.cuda.synchronize()
        clocks, runs = [], []
        for _ in range(args.reps):
            ops.IGEMM_PROFILE = []
            fwd()
            torch.cuda.synchronize()
            q = gpu_query("clocks.sm")
            if q:
                clocks.append(int(float(q[0])))
            runs.append([p["ev"][0].elapsed_time(p["ev"][1]) for p in ops.IGEMM_PROFILE])
            prof = ops.IGEMM_PROFILE
            ops.IGEMM_PROFILE = None
    sms = _lib.load().aab_num_sms()
    med = [sorted(r[i] for r in runs)[len(runs) // 2] for i in range(len(prof))]
    rows = collections.OrderedDict()
    for p, ms in zip(prof, med):
        n_out = p["n"] // 2 if p["geglu"] else p["n"]
        w_out = p["block_n"] // 2 if p["geglu"] else p["block_n"]
        flavour = "geglu" if p["geglu"] else ("16-bit+res" if p["residual"] else "16-bit")
        key = (p["rows"], p["n"], p["k"], p["taps"], p["block_n"], flavour)
        e = rows.setdefault(key, {"launches": 0, "ms": 0.0, "flops": 0.0, "n_out": n_out, "w_out": w_out,
                                  "res": p["residual"]})
        e["launches"] += 1
        e["ms"] += ms
        e["flops"] += p["flops"]
    total = sum(e["ms"] for e in rows.values())
    name = gpu_query("name,power.limit,clocks.max.sm")
    clocks.sort()
    print(f"# {' | '.join(name) if name else torch.cuda.get_device_name(0)} (name | power limit W | max SM MHz); "
          f"median SM clock {clocks[len(clocks) // 2] if clocks else 'n/a'} MHz; {sms} SMs; "
          f"{len(prof)} launches, {total:.1f} ms, {sum(e['flops'] for e in rows.values()) / total / 1e9:.0f} TFLOP/s useful")
    print("| rows | n | k | taps | width | epilogue | launches | ms | share | TFLOP/s | m x n tiles | waves | useful/issued cols "
          "| bound ms | bound by |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for (r, n, k, taps, bn, flavour), e in sorted(rows.items(), key=lambda kv: -kv[1]["ms"]):
        m_tiles = -(-r // 128)
        n_tiles = -(-e["n_out"] // e["w_out"])
        issued = n_tiles * bn
        per = e["flops"] / e["launches"]
        t_mma = per * issued / n / (PEAK_TFLOPS * 1e12)
        byts = 2.0 * (r * k + n * k + r * e["n_out"] * (2 if e["res"] else 1))
        t_mem = byts / (PEAK_TBS * 1e12)
        bound = max(t_mma, t_mem) * 1e3 * e["launches"]
        print(f"| {r} | {n} | {k} | {taps} | {bn} | {flavour} | {e['launches']} | {e['ms']:.2f} | {100 * e['ms'] / total:.1f} % | "
              f"{e['flops'] / e['ms'] / 1e9:.0f} | {m_tiles} x {n_tiles} | {m_tiles * n_tiles / sms:.2f} | {n}/{issued} | "
              f"{bound:.2f} | {'tensor' if t_mma >= t_mem else 'HBM'} |")


if __name__ == "__main__":
    main()
