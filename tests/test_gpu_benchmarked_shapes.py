"""Parity at the shape and dtype that `bench.py` times (BASELINE config 2: CFG batch 2, 16+1 frames, 64x64 latents,
text [2,77,1024], bf16; full-size UNet3D and the full-size SD VAE), against fixtures produced by the VERBATIM reference
files (`tests/golden/make_golden.py benchmarked`: fp32 math on bf16-rounded weights and inputs).

Per stage (conv_in, transformer_in, every down/mid/up block) and for the final output the error of the sm_90a path
against the fp32 oracle is ASSERTED against the yard-stick — the stock PyTorch bf16 execution (cuDNN/cuBLAS/SDPA) of the
same op sequence on the same GPU — and every number goes into the table printed at the end of the test log."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from util import assert_vs_stock, record_parity  # noqa: E402

pytestmark = pytest.mark.gpu

STAGES = (["conv_in2", "transformer_in"] + [f"down_blocks.{i}" for i in range(4)] + ["mid_block"] +
          [f"up_blocks.{i}" for i in range(4)])


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _hook_stages(model, store):
    hooks = []

    def mk(name):
        def hook(mod, args, out):
            o = out[0] if isinstance(out, tuple) else out
            store[name] = (o.sample if hasattr(o, "sample") else o).detach().float()
        return hook
    for name in STAGES:
        hooks.append(model.get_submodule(name).register_forward_hook(mk(name)))
    return hooks


def test_unet_config2_bf16_forward_and_stages():
    from test_gpu_unet import _inputs, _models, _to_nchw
    _no_tf32()
    gold = torch.load(os.path.join(HERE, "golden", "unet_config2_ref.pt"), map_location="cpu")
    dtype = torch.bfloat16
    sh = gold["shape"]
    assert (sh["b"], sh["f"], sh["hw"]) == (2, 16, 64) and gold["dtype"] == "bf16"
    oracle, ours = _models(dict(gold["config"]), dtype)
    inp = _inputs(sh["b"], sh["f"], sh["hw"], sh["lk"], sh["cdim"], dtype)
    mot = torch.tensor([gold["motion"]], device="cuda")
    t = gold["timestep"]
    # the fixture keeps every `out_stride`-th element of the flattened output (and the mean |out| of all of it)
    stride = gold["out_stride"]
    ref = gold["out_sampled"].cuda()
    scale = gold["out_abs_mean"]
    st32, st16 = {}, {}
    hooks = _hook_stages(oracle, st32)
    with torch.no_grad():
        o32 = oracle(inp["sample"].float(), t, inp["ehs"].float(), inp["cond"].float(), inp["mask"].float(), motion=mot)
    for h in hooks:
        h.remove()
    assert tuple(o32.shape) == gold["out_shape"]
    e_or = (o32.reshape(-1)[::stride] - ref).abs().max().item()
    # the oracle restatement on the GPU (fp32, TF32 off) must reproduce the CPU output of the verbatim reference files
    assert e_or <= 5e-3 * scale, f"fp32 oracle on GPU vs verbatim-reference golden: {e_or:.3e} (|ref| {scale:.3e})"
    ours.__dict__["_trace"] = []
    out = ours(inp["sample"], t, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot).sample
    torch.cuda.synchronize()
    trace = ours.__dict__["_trace"]
    ours.__dict__["_trace"] = None
    hooks = _hook_stages(oracle, st16)
    with torch.no_grad():
        stock = oracle.to(dtype)(inp["sample"], t, inp["ehs"], inp["cond"], inp["mask"], motion=mot).float()
    for h in hooks:
        h.remove()
    assert torch.isfinite(out).all()
    case = "unet config2 bf16 [2,4,16,64,64]"
    seen = set()
    for name, x, g in trace:
        key = "conv_in2" if name == "conv_in" else name
        if key not in st32:
            continue
        seen.add(key)
        row = record_parity(case, key, _to_nchw(x, g), st32[key], st16[key])
        # per-stage bar: bf16 chains of different kernel stacks decorrelate, so allow 2x the stock mean error per stage
        assert_vs_stock(row, mean_factor=2.0, max_factor=3.0, mean_floor=1e-3, max_floor=1e-2)
    assert seen == set(STAGES), f"stages not traced: {set(STAGES) - seen}"
    row = record_parity(case, "output (golden)", out.reshape(-1)[::stride], ref, stock.reshape(-1)[::stride])
    assert_vs_stock(row)


def test_vae_fullsize_bf16_encode_decode():
    """Full-size SD VAE (128/256/512/512, mid-block attention at L=4096 d=512, 128ch x 512^2 level) against the
    verbatim reference's `tensor_to_vae_latent` / `decode_latents` outputs."""
    from oracle.composition import AutoencoderKL as OVAE, fill_deterministic, oracle_decode_latents, oracle_encode_image
    from animate_anything_b200.autoencoder_kl import AutoencoderKL
    from animate_anything_b200.common import tensor_to_vae_latent
    from animate_anything_b200.pipeline import tensor2vid
    _no_tf32()
    gold = torch.load(os.path.join(HERE, "golden", "vae_fullsize_ref.pt"), map_location="cpu")
    dtype = torch.bfloat16
    ovae = fill_deterministic(OVAE().eval(), seed=1)
    sd16 = {k: v.to(dtype) for k, v in ovae.state_dict().items()}
    ovae.load_state_dict({k: v.float() for k, v in sd16.items()})
    vae = AutoencoderKL().eval()
    vae.load_state_dict(sd16, strict=True)
    ovae, vae = ovae.cuda(), vae.to(dtype).cuda()
    g = torch.Generator().manual_seed(gold["seed"])
    frames = torch.randn(1, 1, 3, 512, 512, generator=g).clamp(-1, 1).to(dtype).cuda()
    lat = torch.randn(1, 4, 2, 64, 64, generator=g).to(dtype).cuda()
    ref_enc = gold["enc_latents"].cuda()
    vstride = gold["video_stride"]
    ref_vid = gold["video_f16_sampled"].float().cuda()          # every `video_stride`-th element of the flattened video
    with torch.no_grad():
        o_enc = oracle_encode_image(ovae, frames.float())
        o_vid = oracle_decode_latents(ovae, lat.float())
    # oracle on the GPU reproduces the verbatim-reference fixtures (video stored in fp16: 5e-4 relative rounding)
    assert (o_enc - ref_enc).abs().max().item() <= 5e-3 * ref_enc.abs().mean().item()
    assert tuple(o_vid.shape) == gold["video_shape"]
    o_vs = o_vid.reshape(-1)[::vstride]
    assert (o_vs - ref_vid).abs().max().item() <= 5e-3 * ref_vid.abs().mean().item() + 1e-3 * gold["video_abs_max"]
    assert abs(o_vid.abs().mean().item() - gold["video_abs_mean"]) <= 1e-3 * gold["video_abs_mean"]
    enc = tensor_to_vae_latent(frames, vae)
    vid = vae.decode_video(lat)
    u8 = vae.decode_frames_uint8(lat)
    torch.cuda.synchronize()
    with torch.no_grad():
        ovae16 = ovae.to(dtype)
        s_enc = oracle_encode_image(ovae16, frames).float()
        s_vid = oracle_decode_latents(ovae16, lat)
    assert enc.shape == ref_enc.shape and vid.shape == o_vid.shape and vid.dtype == torch.float32
    case = "SD VAE full size bf16"
    assert_vs_stock(record_parity(case, "encode 1x512^2", enc, o_enc, s_enc), max_factor=2.5)
    assert_vs_stock(record_parity(case, "decode 2x512^2", vid, o_vid, s_vid), max_factor=2.5)
    # fused uint8 tail == tensor2vid of the float video, bit for bit
    t2v = tensor2vid(vid.clone())
    assert all((torch.from_numpy(t2v[i]).cuda() == u8[i]).all() for i in range(len(t2v)))
