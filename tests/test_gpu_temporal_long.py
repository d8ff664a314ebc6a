"""GPU: temporal attention for clips of 33..128 frames (the long-clip kernel, bit 1 of `aab_temporal_attn_d64`'s is_bf16)
against float64 softmax attention, and both UNets, the SVD text pipeline and the temporal implicit GEMM at those lengths
against the fp32 oracle and the stock 16-bit torch execution."""
import ctypes as C
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from util import assert_vs_stock, check, record_parity  # noqa: E402
from test_gpu_attention_edges import TOL, _pattern, _rand, _ref  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]


def _reference(qkv, b, t, hw, heads, col0=0):
    """float64 attention over t for every (b, pixel, head); q / k / v at columns col0 + {0, 1, 2} * heads * 64."""
    c = heads * 64
    x = qkv[:, col0:col0 + 3 * c].reshape(b, t, hw, 3, heads, 64).permute(3, 0, 2, 4, 1, 5).reshape(3, b * hw, heads, t, 64)
    return _ref(x[0], x[1], x[2], 0.125).reshape(b, hw, heads, t, 64).permute(0, 3, 1, 2, 4).reshape(b * t * hw, c)


def _long(qkv, b, t, hw, heads, col0=0):
    from animate_anything_b200 import ops
    c = heads * 64
    out = ops.temporal_attn_long(qkv, b, t, hw, heads, col0, col0 + c, col0 + 2 * c)
    torch.cuda.synchronize()
    return out, _reference(qkv, b, t, hw, heads, col0)


# ---------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("t", [1, 2, 17, 32, 33, 47, 48, 49, 63, 64, 65, 78, 79, 96, 127, 128])
def test_long_frame_counts(dtype, t):
    b, hw, heads = 2, 37, 2 + t % 2
    qkv = _rand((b * t * hw, 3 * heads * 64), dtype, 100 + t, 1.5)
    out, ref = _long(qkv, b, t, hw, heads)
    check(f"temporal long t{t} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("t", [33, 78, 128])
@pytest.mark.parametrize("pattern", ["max_first", "max_last", "onehot_last"])
def test_long_large_logits(dtype, t, pattern):
    b, hw, heads = 2, 41, 2
    c = heads * 64
    qkv = _rand((b * t * hw, 3 * c), dtype, t)
    v = qkv.view(b, t, hw, 3, heads, 64)
    v[:, :, :, 0, :, 0] = 4.0
    v[:, :, :, 1, :, 0] = _pattern(pattern, t, t).to(dtype).view(1, t, 1, 1)
    out, ref = _long(qkv, b, t, hw, heads)
    check(f"temporal long {pattern} t{t} {dtype}", out, ref, *TOL[dtype])


def _persistent_shape(t):
    """(b, t, hw, heads) with at least three items per CTA of the persistent grid (one item per CTA at a time, four CTAs per
    SM up to 64 frames, two above): every CTA reuses both buffers, and the last round is ragged."""
    from animate_anything_b200 import _lib
    b, hw, heads = 2, 1000, 2
    total = b * hw * heads
    stride = min(total, (4 if t <= 64 else 2) * _lib.load().aab_num_sms())
    assert total >= 3 * stride and total % stride != 0, (total, stride)
    return b, t, hw, heads


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("t", [49, 78])
def test_long_persistent_loop(dtype, t):
    b, t, hw, heads = _persistent_shape(t)
    qkv = _rand((b * t * hw, 3 * heads * 64), dtype, 7)
    out, ref = _long(qkv, b, t, hw, heads)
    check(f"temporal long persistent b{b} t{t} hw{hw} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("heads", [5, 10, 20])
def test_long_fused_qkv_row_layout(dtype, heads):
    """The UNet's layout: q | k | v column blocks of one fused row, here behind 40 leading columns and before 24 more."""
    b, t, hw = 2, 78, 12
    c = heads * 64
    qkv = _rand((b * t * hw, 40 + 3 * c + 24), dtype, heads)
    out, ref = _long(qkv, b, t, hw, heads, col0=40)
    check(f"temporal long fused row heads{heads} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
def test_long_output_stays_in_its_columns(dtype):
    """Output rows wider than heads x 64, written from column 16 on: every column outside the heads keeps its sentinel."""
    from animate_anything_b200 import _lib
    b, t, hw, heads = 2, 78, 9, 2
    c = heads * 64
    qkv = _rand((b * t * hw, 3 * c), dtype, 3)
    ld_out = c + 48
    sentinel = -1234.0
    out = torch.full((b * t * hw, ld_out), sentinel, device="cuda", dtype=dtype)
    bf = (1 if dtype == torch.bfloat16 else 0) | 2
    r = _lib.load().aab_temporal_attn_d64(C.c_void_p(qkv.data_ptr()), qkv.stride(0), 0, c, 2 * c,
                                          C.c_void_p(out.data_ptr() + 16 * out.element_size()), ld_out, b, t, hw, heads,
                                          0.125, bf, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert r == 0
    torch.cuda.synchronize()
    ref = _reference(qkv, b, t, hw, heads)
    check(f"temporal long strided out {dtype}", out[:, 16:16 + c], ref, *TOL[dtype])
    assert (out[:, :16] == sentinel).all() and (out[:, 16 + c:] == sentinel).all()


def test_long_argument_checks():
    from animate_anything_b200 import _lib
    lib = _lib.load()
    qkv = torch.zeros((130 * 4, 3 * 64), device="cuda", dtype=torch.float16)
    out = torch.zeros((130 * 4, 64), device="cuda", dtype=torch.float16)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def ta(t, flags):
        return lib.aab_temporal_attn_d64(C.c_void_p(qkv.data_ptr()), 192, 0, 64, 128, C.c_void_p(out.data_ptr()), 64, 1, t, 4,
                                         1, 0.125, flags, stream)
    assert ta(129, 2) == 1 and ta(129, 3) == 1 and ta(0, 2) == 1 and ta(0, 3) == 1
    for flags in (4, 5, 6, 7, 8, 10, -1, 1 << 30):
        assert ta(33, flags) == 1, flags
    assert ta(33, 0) == 1 and ta(33, 1) == 1                   # without bit 1: the v2 kernel's 32-frame limit
    assert ta(33, 2) == 0 and ta(128, 3) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- temporal implicit GEMM
@pytest.mark.parametrize("dtype", DTYPES)
def test_tconv3_79_frames(dtype):
    from animate_anything_b200 import ops
    igemm_tol = {torch.float16: (1e-3, 1e-4), torch.bfloat16: (8e-3, 8e-4)}       # as tests/test_gpu_igemm.py
    b, t, hw, c = 2, 79, 40, 128
    x = _rand((b * t * hw, c), dtype, 1)
    wt = _rand((c, c, 3, 1, 1), dtype, 2, (3 * c) ** -0.5)
    bias = _rand((c,), torch.float32, 3)
    res = _rand((b * t * hw, c), dtype, 4)
    x5 = x.float().reshape(b, t, hw, 1, c).permute(0, 4, 1, 2, 3)
    ref = F.conv3d(x5, wt.float(), bias, padding=(1, 0, 0)).permute(0, 2, 3, 4, 1).reshape(-1, c) + res.float()
    wp = wt.reshape(c, c, 3).permute(0, 2, 1).reshape(c, 3 * c).contiguous()
    out = ops.tconv3(x, b, t, hw, wp, bias, residual=res)
    torch.cuda.synchronize()
    check(f"tconv3 b{b} t{t} hw{hw} c{c} {dtype}", out, ref, *igemm_tol[dtype])


# ---------------------------------------------------------------------------------------------- UNet3D
@pytest.mark.parametrize("dtype", DTYPES)
def test_unet3d_forward_48_frames(dtype):
    """LatentToVideoPipeline(num_frames=48) runs the UNet on 49 frames (48 + the condition frame)."""
    from test_gpu_unet import SMALL, _run_case
    _run_case(SMALL, dtype, b=2, f=48, hw=16, lk=77)


# ---------------------------------------------------------------------------------------------- SVD UNet
def _svd_inputs(nf, dtype, seed=3):
    g = torch.Generator().manual_seed(seed)
    h, w = 16, 24
    lat = torch.randn(1, nf, 4, h, w, generator=g)
    il = torch.randn(1, nf, 4, h, w, generator=g)
    mask = (torch.rand(1, 1, 1, h, w, generator=g) > 0.5).float().expand(2, nf, 1, h, w)
    x = torch.cat([mask, torch.cat([lat, lat]), torch.cat([torch.zeros_like(il), il])], dim=2).to(dtype).cuda()
    emb = torch.randn(1, 1, 96, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb]).to(dtype).cuda()
    ids = torch.tensor([[6.0, 127.0, 0.02]] * 2).cuda()
    return x, ehs, ids


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nf", [40, 78])
def test_svd_unet_forward_long_clip(dtype, nf):
    from test_gpu_svd import _pair
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _pair(dtype)
    x, ehs, ids = _svd_inputs(nf, dtype)
    t = torch.tensor(1.6378)
    with torch.no_grad():
        ref = oracle(x.float(), t, ehs.float(), ids, return_dict=False)[0]
    out = ours(x, t, ehs, ids).sample
    torch.cuda.synchronize()
    with torch.no_grad():
        stock = oracle.to(dtype)(x, t, ehs, ids.to(dtype), return_dict=False)[0].float()
    assert out.shape == ref.shape == (2, nf, 4, 16, 24) and torch.isfinite(out).all()
    assert_vs_stock(record_parity(f"SVD UNet small {str(dtype).split('.')[-1]} F={nf}", "output", out, ref, stock))


# ---------------------------------------------------------------------------------------------- SVD text pipeline, 78 frames
def test_svd_text_pipeline_78_frames_as_the_app_calls_it():
    """`TextStableVideoDiffusionPipeline.__call__` called unbound with the pipeline as first argument, as app_svd.py:120-133
    calls the reference's: 78 frames (the app's maximum), per-frame mask with frame 0 cleared, caller-supplied
    `condition_latent`, decode_chunk_size 7; latents and decoded frames against the oracle loop."""
    from oracle.composition import EulerDiscreteScheduler as OEuler, SVD_SCHED, oracle_svd_sampling_loop
    from animate_anything_b200.pipeline_svd import TextStableVideoDiffusionPipeline
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    from test_gpu_svd import _pair, _vae_pair
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dtype = torch.float16
    nf = 78
    ounet, unet = _pair(dtype)
    ovae, vae = _vae_pair(dtype)
    g = torch.Generator().manual_seed(9)
    img = torch.randn(1, 3, 128, 192, generator=g).clamp(-1, 1)
    mask = (torch.rand(1, nf, 1, 16, 24, generator=g) > 0.5).float()
    mask[:, 0] = 0
    lat0 = torch.randn(1, nf, 4, 16, 24, generator=g)
    cl = torch.randn(1, nf, 4, 16, 24, generator=g)
    emb = torch.randn(1, 1, 96, generator=g)
    pipe = TextStableVideoDiffusionPipeline(vae=vae, image_encoder=None, unet=unet, scheduler=EulerDiscreteScheduler(**SVD_SCHED))
    kw = dict(image=img, width=192, height=128, num_frames=nf, num_inference_steps=3, decode_chunk_size=7, mask=mask,
              condition_type="image", condition_latent=cl, noise_aug_strength=0.0, latents=lat0, image_embeddings=emb,
              return_dict=False)
    lat = TextStableVideoDiffusionPipeline.__call__(pipe, output_type="latent", **kw)
    frames = TextStableVideoDiffusionPipeline.__call__(pipe, output_type="pt", **kw)
    torch.cuda.synchronize()
    okw = dict(num_inference_steps=3, noise_aug_strength=0.0, decode_chunk_size=7)
    with torch.no_grad():
        il32 = ovae.encode(img.to(dtype).float().cuda()).latent_dist.mode()
        rf, rl = oracle_svd_sampling_loop(ounet, OEuler(**SVD_SCHED), ovae, emb.to(dtype).float().cuda(), il32, None,
                                          lat0.to(dtype).float().cuda(), frame_mask=mask.cuda(),
                                          condition_latent=cl.to(dtype).float().cuda(), **okw)
        o16u, o16v = ounet.to(dtype), ovae.to(dtype)
        il16 = o16v.encode(img.to(dtype).cuda()).latent_dist.mode()
        sf, sl = oracle_svd_sampling_loop(o16u, OEuler(**SVD_SCHED), o16v, emb.to(dtype).cuda(), il16, None,
                                          lat0.to(dtype).cuda(), frame_mask=mask.to(dtype).cuda(),
                                          condition_latent=cl.to(dtype).cuda(), **okw)
    assert lat.shape == rl.shape == (1, nf, 4, 16, 24)
    case = "SVD Text pipeline fp16 78 frames"
    assert_vs_stock(record_parity(case, "latents", lat, rl, sl), mean_factor=3.0, max_factor=4.0, mean_floor=5e-4,
                    max_floor=5e-3)
    got = frames[0]                                         # [F, 3, H, W] in [0, 1]
    want = (rf[0].permute(1, 0, 2, 3) / 2 + 0.5).clamp(0, 1)
    stock = (sf[0].permute(1, 0, 2, 3) / 2 + 0.5).clamp(0, 1)
    assert got.shape == want.shape == (nf, 3, 128, 192)
    assert_vs_stock(record_parity(case, "frames", got, want, stock), mean_factor=3.0, max_factor=4.0, mean_floor=2e-3,
                    max_floor=2e-2)


# ---------------------------------------------------------------------------------------------- more than 128 frames
def _cuda_kernels_during(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        with pytest.raises(NotImplementedError, match="128 frames"):
            fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_more_than_128_frames_fail_before_any_launch():
    from test_gpu_svd import _pair
    from test_gpu_unet import SMALL, _inputs, _models
    _, unet3d = _models(SMALL, torch.float16)
    inp = _inputs(1, 128, 16, 77, SMALL["cross_attention_dim"], torch.float16)       # 128 frames + condition = 129
    mot = torch.tensor([4.0], device="cuda")
    ran = _cuda_kernels_during(lambda: unet3d(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"],
                                              motion=mot))
    assert not ran, ran[:10]
    _, svd = _pair(torch.float16)
    x, ehs, ids = _svd_inputs(129, torch.float16)
    t = torch.tensor(1.6378)
    ran = _cuda_kernels_during(lambda: svd(x, t, ehs, ids))
    assert not ran, ran[:10]
