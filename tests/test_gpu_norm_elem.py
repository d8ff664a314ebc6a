"""GPU parity of the normalisation / elementwise / boundary kernels vs plain PyTorch fp32."""
import math

import pytest
import torch
import torch.nn.functional as F

from util import check

pytestmark = pytest.mark.gpu
# fp16: the north-star tolerance (rtol=1e-3, atol=1e-4); bf16 8x looser
TOL = {torch.float16: (1e-3, 1e-4), torch.bfloat16: (8e-3, 8e-4)}


def _rand(shape, dtype, scale=1.0, seed=0, shift=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale + shift).to(dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("samples,rows,c,silu", [(4, 256, 320, True), (2, 17 * 64, 640, False), (3, 100, 1280, True),
                                                 (2, 4096, 128, True), (1, 64, 1920, True)])
def test_groupnorm(dtype, samples, rows, c, silu):
    from animate_anything_b200 import ops
    x = _rand((samples * rows, c), dtype, 1.5, 1, shift=0.3)
    gamma = _rand((c,), torch.float32, 0.2, 2, shift=1.0)
    beta = _rand((c,), torch.float32, 0.2, 3)
    y = ops.groupnorm(x, samples, rows, gamma, beta, 1e-5, silu)
    xr = x.float().reshape(samples, rows, c).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, gamma, beta, 1e-5)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(samples * rows, c)
    check(f"groupnorm s{samples} r{rows} c{c} {dtype}", y, ref, *TOL[dtype])


@pytest.mark.parametrize("samples,rows,c", [(34, 4096, 320), (2, 69632, 320), (2, 1088, 1280), (34, 64, 2560)])
def test_groupnorm_benchmarked_shapes_and_repeat(samples, rows, c):
    """The extents of a config-2 UNet forward (2-D per frame, 3-D per clip) through ONE shared workspace: the tickets must
    come back to zero and must not alias another call's statistics (fixed header), so a SECOND call gives the same bits."""
    from animate_anything_b200 import ops
    dtype = torch.bfloat16
    x = _rand((samples * rows, c), dtype, 1.5, 1, shift=0.3)
    gamma = _rand((c,), torch.float32, 0.2, 2, shift=1.0)
    beta = _rand((c,), torch.float32, 0.2, 3)
    y1 = ops.groupnorm(x, samples, rows, gamma, beta, 1e-5, True)
    y2 = ops.groupnorm(x, samples, rows, gamma, beta, 1e-5, True)
    assert torch.equal(y1, y2)
    xr = x.float().reshape(samples, rows, c).permute(0, 2, 1)
    ref = F.silu(F.group_norm(xr, 32, gamma, beta, 1e-5)).permute(0, 2, 1).reshape(samples * rows, c)
    check(f"groupnorm s{samples} r{rows} c{c}", y1, ref, *TOL[dtype])


def test_groupnorm_large_mean_no_cancellation():
    """Statistics are E[x^2] - E[x]^2 from fp32 per-thread partials combined in fp64: a mean 50x the standard deviation
    must not lose the variance (VERDICT r1 weak 17)."""
    from animate_anything_b200 import ops
    dtype = torch.float16
    samples, rows, c = 2, 4096, 320
    x = _rand((samples * rows, c), dtype, 1.0, 7, shift=50.0)
    gamma = torch.ones(c, device="cuda")
    beta = torch.zeros(c, device="cuda")
    y = ops.groupnorm(x, samples, rows, gamma, beta, 1e-5, False)
    xr = x.double().reshape(samples, rows, c).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, gamma.double(), beta.double(), 1e-5).permute(0, 2, 1).reshape(samples * rows, c)
    check("groupnorm mean=50 std=1", y, ref.float(), 2e-3, 2e-3)


def test_groupnorm_batch_invariant():
    """A sample's output does not depend on the batch it is normalised in (fixed (rows, C) row partition)."""
    from animate_anything_b200 import ops
    x = _rand((4 * 1088, 320), torch.float16, 1.5, 5, shift=0.3)
    gamma = _rand((320,), torch.float32, 0.2, 2, shift=1.0)
    beta = _rand((320,), torch.float32, 0.2, 3)
    full = ops.groupnorm(x, 4, 1088, gamma, beta, 1e-5, True)
    one = ops.groupnorm(x[2 * 1088:3 * 1088].contiguous(), 1, 1088, gamma, beta, 1e-5, True)
    assert torch.equal(full[2 * 1088:3 * 1088], one)


def test_groupnorm_concat():
    from animate_anything_b200 import ops
    dtype = torch.float16
    samples, rows, c1, c2 = 3, 256, 1280, 640
    x1 = _rand((samples * rows, c1), dtype, 1.0, 1)
    x2 = _rand((samples * rows, c2), dtype, 2.0, 2, shift=-0.5)
    gamma = _rand((c1 + c2,), torch.float32, 0.2, 3, shift=1.0)
    beta = _rand((c1 + c2,), torch.float32, 0.2, 4)
    y = ops.groupnorm(x1, samples, rows, gamma, beta, 1e-5, True, x2=x2)
    xc = torch.cat([x1, x2], dim=1).float().reshape(samples, rows, c1 + c2).permute(0, 2, 1)
    ref = F.silu(F.group_norm(xc, 32, gamma, beta, 1e-5)).permute(0, 2, 1).reshape(samples * rows, c1 + c2)
    check("groupnorm virtual concat 1280+640", y, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rows,c", [(1000, 320), (77, 1280), (4096, 512), (10, 640)])
def test_layernorm(dtype, rows, c):
    from animate_anything_b200 import ops
    x = _rand((rows, c), dtype, 2.0, 1, shift=0.5)
    gamma = _rand((c,), torch.float32, 0.2, 2, shift=1.0)
    beta = _rand((c,), torch.float32, 0.2, 3)
    y = ops.layernorm(x, gamma, beta, 1e-5)
    ref = F.layer_norm(x.float(), (c,), gamma, beta, 1e-5)
    check(f"layernorm {rows}x{c} {dtype}", y, ref, *TOL[dtype])


def test_softmax_rows_and_transpose():
    from animate_anything_b200 import ops
    s = _rand((300, 1000), torch.float32, 3.0, 1)
    p = ops.softmax_rows(s, torch.float16)
    check("softmax rows", p, torch.softmax(s, dim=-1), 1e-3, 1e-5)
    src = _rand((3 * 100, 96), torch.float16, 1.0, 2)
    dst = ops.transpose_batched(src, 32, 3, 100, 64)
    ref = src[:, 32:96].reshape(3, 100, 64).permute(0, 2, 1)
    assert torch.equal(dst, ref.contiguous())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_unet_boundary_kernels(dtype):
    from animate_anything_b200 import ops
    b, f, h, w = 2, 5, 8, 16
    sample = _rand((1, 4, f, h, w), dtype, 1.0, 1).expand(b, 4, f, h, w)      # batch-stride-0 view (CFG duplicate)
    cond = _rand((b, 4, 1, h, w), dtype, 1.0, 2)
    mask = (_rand((1, 1, 1, h, w), torch.float32, 1.0, 3) > 0).to(dtype)
    out = ops.unet_in_assemble(sample, cond, mask, f + 1)
    full = torch.cat([cond, sample], dim=2)                                      # b 4 T h w
    m = mask.expand(b, 1, f + 1, h, w)
    ref = torch.cat([m, full], dim=1).permute(0, 2, 3, 4, 1)                     # b T h w 5
    assert torch.equal(out[..., :5], ref.contiguous())
    assert torch.all(out[..., 5:] == 0)
    out2 = ops.unet_in_assemble(sample, cond, None, f + 1)
    assert torch.equal(out2[..., :4], full.permute(0, 2, 3, 4, 1).contiguous())
    # output finalize
    y = _rand((b * (f + 1) * h * w, 4), torch.float32, 1.0, 4)
    o = ops.unet_out_finalize(y, b, f + 1, h, w, dtype)
    ref = y.reshape(b, f + 1, h, w, 4).permute(0, 4, 1, 2, 3)[:, :, 1:].to(dtype)
    assert torch.equal(o, ref.contiguous())
    # timestep embedding
    t = torch.tensor([981.0], device="cuda")
    e = ops.timestep_embed(t, b, 320, dtype)
    half = 160
    freq = torch.exp(-math.log(10000) * torch.arange(half, device="cuda", dtype=torch.float32) / half)
    a = t[:, None] * freq[None]
    ref = torch.cat([torch.cos(a), torch.sin(a)], dim=-1).expand(b, 320)
    check(f"timestep embed {dtype}", e, ref, *TOL[dtype])
    # geglu + upsample
    x = _rand((100, 256), dtype, 1.0, 5)
    g = ops.geglu(x)
    check("geglu", g, x[:, :128].float() * F.gelu(x[:, 128:].float()), *TOL[dtype])
    xi = _rand((3, 4, 6, 16), dtype, 1.0, 6)
    up = ops.upsample2x(xi)
    ref = F.interpolate(xi.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1).to(dtype)
    assert torch.equal(up, ref.contiguous())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_cfg_scheduler_step(dtype):
    from animate_anything_b200 import ops
    n, f, h, w = 1, 4, 8, 8
    t = f + 1
    eps = _rand((2 * n * t * h * w, 4), torch.float32, 1.0, 1)
    x = _rand((n, 4, f, h, w), dtype, 1.0, 2)
    hist = _rand((n, 4, f, h, w), torch.float32, 1.0, 3)
    hist0 = hist.clone()
    coef = torch.tensor([[0.0] * 6, [1.1, -0.3, 0.7, 0.2, -0.4, 0.15]], device="cuda", dtype=torch.float32)
    step = torch.tensor([1], device="cuda", dtype=torch.int32)
    out = torch.empty_like(x)
    ops.cfg_scheduler_step(eps, 4, True, 9.0, x, out, hist, coef, step)
    e = eps.reshape(2 * n, t, h, w, 4).permute(0, 4, 1, 2, 3)[:, :, 1:]
    e = e[:n] + 9.0 * (e[n:] - e[:n])
    k = coef[1]
    x0 = k[0] * x.float() + k[1] * e
    ref = k[2] * x.float() + k[3] * e + k[4] * x0 + k[5] * hist0
    check(f"cfg+scheduler step {dtype}", out, ref, *TOL[dtype])
    check("x0 history", hist, x0, 1e-5, 1e-5)


def test_vae_boundary_kernels():
    from animate_anything_b200 import ops
    dtype = torch.float16
    img = _rand((2, 3, 16, 24), dtype, 1.0, 1)
    o = ops.image_to_nhwc8(img)
    assert torch.equal(o[..., :3], img.permute(0, 2, 3, 1).contiguous()) and torch.all(o[..., 3:] == 0)
    b, f, h, w = 1, 3, 8, 8
    mom = _rand((b * f * h * w, 8), dtype, 1.0, 2)
    wq = _rand((8, 8), torch.float32, 0.3, 3)
    bq = _rand((8,), torch.float32, 0.3, 4)
    lat = ops.vae_enc_finalize(mom, wq, bq, 1.0, b, f, h, w)
    ref = (mom.float() @ wq.t() + bq).reshape(b, f, h, w, 8).permute(0, 4, 1, 2, 3)
    check("vae enc finalize", lat, ref, 1e-3, 1e-3)
    latents = _rand((b, 4, f, h, w), dtype, 1.0, 5)
    wp = _rand((4, 4), torch.float32, 0.5, 6)
    bp = _rand((4,), torch.float32, 0.5, 7)
    z = ops.vae_dec_in(latents, 1 / 0.18215, wp, bp)
    zr = (latents.float() / 0.18215).to(dtype).float().permute(0, 2, 3, 4, 1).reshape(-1, 4) @ wp.t() + bp
    check("vae dec in", z.reshape(-1, 8)[:, :4], zr, 2e-3, 2e-3)
    y = _rand((b * f * 16 * 16, 16), torch.float32, 1.0, 8)
    vid = ops.vae_dec_finalize(y, b, f, 16, 16, False)
    ref = y[:, :3].to(dtype).float().reshape(b, f, 16, 16, 3).permute(0, 4, 1, 2, 3)
    assert torch.equal(vid, ref.contiguous())


def _producer(ops, x, w, bias, mode, res=None, **kw):
    if mode == "linear":
        return ops.linear(x, w, bias, residual=res, stats=True, **kw)
    return ops.conv3x3(x, w, bias, residual=res, stats=True, **kw)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mode,m_or_shape,k,n,bn", [("linear", 1024, 320, 320, 64), ("linear", 4352, 640, 640, 128),
                                                     ("linear", 2048, 1280, 1280, 256), ("conv", (3, 32, 32), 320, 320, 128),
                                                     ("conv", (2, 16, 16), 640, 1280, 256)])
def test_igemm_epilogue_column_statistics(dtype, mode, m_or_shape, k, n, bn):
    """`stats=True`: the epilogue's per-(128-row tile, column) sum / sum of squares of the ROUNDED output it stores."""
    from animate_anything_b200 import ops
    if mode == "linear":
        m = m_or_shape
        x = _rand((m, k), dtype, 1.0, 1)
        w = _rand((n, k), dtype, k ** -0.5, 2)
    else:
        nb, h, wd = m_or_shape
        m = nb * h * wd
        x = _rand((nb, h, wd, k), dtype, 1.0, 1)
        w = _rand((n, 9 * k), dtype, (9 * k) ** -0.5, 2)
    bias = _rand((n,), torch.float32, 1.0, 3)
    res = _rand((m, n), dtype, 1.0, 4)
    out = _producer(ops, x, w, bias, mode, res=res, block_n=bn)
    st = getattr(out, "_aab_stats", None)
    assert st is not None and tuple(st.shape) == (m // 128, n, 2)
    o = out.double().reshape(m // 128, 128, n)
    check(f"colstats sum {mode} {dtype}", st[..., 0], o.sum(1).float(), 1e-5, 1e-3)
    check(f"colstats sumsq {mode} {dtype}", st[..., 1], (o * o).sum(1).float(), 1e-5, 1e-3)
    # an epilogue that cannot emit them (fp32 output) must say so by not attaching anything
    assert getattr(ops.linear(_rand((256, 64), dtype), _rand((64, 64), dtype), None, out_f32=True, stats=True), "_aab_stats", None) is None


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("samples,rows,c,silu", [(4, 256, 320, True), (2, 17 * 256, 640, False), (34, 1024, 640, True)])
def test_groupnorm_from_producer_statistics(dtype, samples, rows, c, silu):
    """GroupNorm fed by the producing GEMM's column statistics == the two-pass GroupNorm of the same tensor up to the
    rounding of fp32 tile sums (well inside the fp32-reference tolerance), second source = virtual concat."""
    from animate_anything_b200 import ops
    m = samples * rows
    x = _rand((m, 320), dtype, 1.0, 1)
    w = _rand((c, 320), dtype, 320 ** -0.5, 2)
    bias = _rand((c,), torch.float32, 0.5, 3)
    h = ops.linear(x, w, bias, stats=True)
    h2 = ops.linear(x, w.flip(0).contiguous(), bias, stats=True)
    assert getattr(h, "_aab_stats", None) is not None
    gamma = _rand((c,), torch.float32, 0.2, 2, shift=1.0)
    beta = _rand((c,), torch.float32, 0.2, 3)
    y = ops.groupnorm(h, samples, rows, gamma, beta, 1e-5, silu)
    y_again = ops.groupnorm(h, samples, rows, gamma, beta, 1e-5, silu)
    assert torch.equal(y, y_again)
    plain = h.clone()                                  # no statistics attached -> two-pass kernel
    y2 = ops.groupnorm(plain, samples, rows, gamma, beta, 1e-5, silu)
    ref = F.group_norm(h.float().reshape(samples, rows, c).permute(0, 2, 1), 32, gamma, beta, 1e-5)
    ref = (F.silu(ref) if silu else ref).permute(0, 2, 1).reshape(m, c)
    check(f"groupnorm(colstats) s{samples} r{rows} c{c} {dtype}", y, ref, *TOL[dtype])
    ulp = 2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7
    assert (y.float() - y2.float()).abs().max().item() <= 2 * ulp * max(1.0, y2.float().abs().max().item())
    # virtual concat of two producers
    g2 = _rand((2 * c,), torch.float32, 0.2, 5, shift=1.0)
    b2 = _rand((2 * c,), torch.float32, 0.2, 6)
    yc = ops.groupnorm(h, samples, rows, g2, b2, 1e-5, silu, x2=h2)
    refc = F.group_norm(torch.cat([h, h2], 1).float().reshape(samples, rows, 2 * c).permute(0, 2, 1), 32, g2, b2, 1e-5)
    refc = (F.silu(refc) if silu else refc).permute(0, 2, 1).reshape(m, 2 * c)
    check(f"groupnorm(colstats, concat) {dtype}", yc, refc, *TOL[dtype])
    # batch invariance: sample 1 alone gives the same bits as inside the batch
    xs = x[rows:2 * rows].contiguous()
    hs = ops.linear(xs, w, bias, stats=True)
    ys = ops.groupnorm(hs, 1, rows, gamma, beta, 1e-5, silu)
    assert torch.equal(ys, y[rows:2 * rows])
