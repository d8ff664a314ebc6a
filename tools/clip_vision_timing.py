"""Times the CLIP ViT-H/14 image tower (clip_vision.CLIPVisionModelWithProjection: 32 layers x 1280, 16 heads of 80,
224 px; random weights) at B = 1 in fp16 with CUDA events after warm-up, next to `transformers` fp16 with SDPA on the same
GPU, and the head-dim-80 flash attention kernel alone at the tower's shape.  Prints the card name and power limit of the
run beside the numbers.  Usage: python tools/clip_vision_timing.py [iters]"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from animate_anything_b200 import ops  # noqa: E402
from animate_anything_b200.clip_vision import CLIPVisionModelWithProjection  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_ms(fn, iters):
    for _ in range(3):
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


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection as HF
    dtype = torch.float16
    cfg = CLIPVisionConfig(hidden_size=1280, intermediate_size=5120, projection_dim=1024, num_hidden_layers=32,
                           num_attention_heads=16, image_size=224, patch_size=14, hidden_act="gelu",
                           attn_implementation="sdpa")
    torch.manual_seed(0)
    hf = HF(cfg).eval().to(dtype).cuda()
    ours = CLIPVisionModelWithProjection.from_hf(hf)
    pv = torch.randn(1, 3, 224, 224, device="cuda", dtype=dtype)
    t_ours = time_ms(lambda: ours(pv), iters)
    with torch.no_grad():
        t_hf = time_ms(lambda: hf(pixel_values=pv), iters)
    l, heads, c = 257, 16, 1280
    qkv = torch.randn(l, 3 * c, device="cuda", dtype=dtype)
    t_fa = time_ms(lambda: ops.flash_attn_d80(qkv, 0, qkv, c, 2 * c, 1, l, l, heads), iters)
    fa_flops = 4.0 * heads * l * l * 80
    name, power = card()
    print(f"card: {name}, power limit {power}")
    print(f"CLIP ViT-H/14 tower, B=1, 224^2, fp16, median of {iters}: sm_90a kernels {t_ours:.3f} ms, "
          f"transformers (SDPA) {t_hf:.3f} ms")
    print(f"flash_attn_d80 [1 x 16 heads x 257 x 257]: {t_fa * 1e3:.1f} us, {fa_flops / t_fa / 1e9:.2f} TFLOP/s")


if __name__ == "__main__":
    main()
