"""GPU parity of the wgmma implicit-GEMM kernel against plain PyTorch fp32 on the same 16-bit-rounded inputs.
Tolerance: the output is rounded once to fp16 (rel 2^-11) / bf16 (rel 2^-8) after fp32 accumulation."""
import pytest
import torch
import torch.nn.functional as F

from util import check

pytestmark = pytest.mark.gpu

# fp16: the north-star tolerance (rtol=1e-3, atol=1e-4).  bf16 has 3 fewer mantissa bits: 8x looser.
TOL = {torch.float16: (1e-3, 1e-4), torch.bfloat16: (8e-3, 8e-4)}


def _ops():
    from animate_anything_b200 import ops
    return ops


def _rand(shape, dtype, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("m,k,n,bn", [(128, 64, 64, 64), (300, 320, 320, 128), (1000, 640, 1280, 256),
                                       (77, 1024, 640, 64), (2, 1280, 320, 128), (4096, 512, 512, 256)])
def test_linear_plain(dtype, m, k, n, bn):
    ops = _ops()
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    ref = x.float() @ w.float().t() + b
    out = ops.linear(x, w, b, block_n=bn)
    torch.cuda.synchronize()
    check(f"linear {m}x{k}x{n} bn{bn} {dtype}", out, ref, *TOL[dtype])
    out2 = ops.linear(x, w, b, block_n=bn, direct=True)
    torch.cuda.synchronize()
    check(f"linear-direct {m}x{k}x{n} bn{bn} {dtype}", out2, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_linear_epilogues(dtype):
    ops = _ops()
    m, k, n = 1500, 320, 640
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    res = _rand((m, n), dtype, 1.0, 4)
    b2 = _rand((3, n), torch.float32, 1.0, 5)
    ref = (x.float() @ w.float().t() + b + b2.repeat_interleave(500, dim=0) + res.float())
    ref_silu = F.silu(ref) * 0.5
    out = ops.linear(x, w, b, bias2=b2, rows_per_bias2=500, residual=res)
    check("linear+bias2+residual", out, ref, *TOL[dtype])
    out = ops.linear(x, w, b, bias2=b2, rows_per_bias2=500, residual=res, act=ops.ACT_SILU, out_scale=0.5)
    check("linear+silu+scale", out, ref_silu, *TOL[dtype])
    out = ops.linear(x, w, b, out_f32=True)
    assert out.dtype == torch.float32
    check("linear f32 out", out, x.float() @ w.float().t() + b, 1e-4, 1e-4)
    # GEGLU: w rows [0,n/2) values, [n/2,n) gates
    full = x.float() @ w.float().t() + b
    ref_g = full[:, : n // 2] * F.gelu(full[:, n // 2:])
    for bn in (128, 256):
        out = ops.linear(x, w, b, geglu=True, block_n=bn)
        check(f"linear geglu bn{bn}", out, ref_g, *TOL[dtype])
    # tiny N (conv_out-like), direct store with masking
    w4 = _rand((4, k), dtype, k ** -0.5, 7)
    out = ops.linear(x, w4, None, out_f32=True)
    check("linear n=4 f32", out, x.float() @ w4.float().t(), 1e-4, 1e-4)


def _conv_weight(cout, cin, dtype, seed):
    return _rand((cout, cin, 3, 3), dtype, (9 * cin) ** -0.5, seed)


def _prep3x3(w):
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nb,h,w,cin,cout", [(2, 16, 16, 64, 64), (3, 8, 8, 128, 320), (1, 64, 64, 64, 128),
                                              (2, 32, 32, 320, 320), (1, 20, 24, 64, 64)])
def test_conv3x3(dtype, nb, h, w, cin, cout):
    ops = _ops()
    x = _rand((nb, h, w, cin), dtype, 1.0, 1)
    wt = _conv_weight(cout, cin, dtype, 2)
    b = _rand((cout,), torch.float32, 1.0, 3)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), b, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    out = ops.conv3x3(x, _prep3x3(wt), b)
    check(f"conv3x3 {nb}x{h}x{w}x{cin}->{cout} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", [torch.float16])
def test_conv3x3_concat_and_temb(dtype):
    ops = _ops()
    nb, h, w, c1, c2, cout = 4, 16, 16, 128, 64, 192
    x1 = _rand((nb, h, w, c1), dtype, 1.0, 1)
    x2 = _rand((nb, h, w, c2), dtype, 1.0, 2)
    wt = _conv_weight(cout, c1 + c2, dtype, 3)
    b = _rand((cout,), torch.float32, 1.0, 4)
    temb = _rand((2, cout), torch.float32, 1.0, 5)     # 2 batch elements x 2 frames each
    xc = torch.cat([x1, x2], dim=-1)
    ref = F.conv2d(xc.float().permute(0, 3, 1, 2), wt.float(), b, padding=1).permute(0, 2, 3, 1)
    ref = ref + temb.repeat_interleave(2, dim=0)[:, None, None, :]
    out = ops.conv3x3(x1, _prep3x3(wt), b, x2=x2, bias2=temb, rows_per_bias2=2 * h * w)
    check("conv3x3 virtual-concat + per-sample bias", out, ref.reshape(-1, cout), *TOL[dtype])
    # 1x1 shortcut over the virtual concat
    w1 = _rand((cout, c1 + c2), dtype, (c1 + c2) ** -0.5, 6)
    ref1 = xc.float().reshape(-1, c1 + c2) @ w1.float().t() + b
    out1 = ops.conv1x1_cat(x1.reshape(-1, c1), x2.reshape(-1, c2), w1, b)
    check("conv1x1 virtual-concat", out1, ref1, *TOL[dtype])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mode", ["sym", "br"])
def test_conv3x3_stride2(dtype, mode):
    ops = _ops()
    nb, h, w, c, cout = 3, 16, 32, 64, 128
    x = _rand((nb, h, w, c), dtype, 1.0, 1)
    wt = _conv_weight(cout, c, dtype, 2)
    b = _rand((cout,), torch.float32, 1.0, 3)
    xin = x.float().permute(0, 3, 1, 2)
    if mode == "sym":
        ref = F.conv2d(xin, wt.float(), b, stride=2, padding=1)
    else:
        ref = F.conv2d(F.pad(xin, (0, 1, 0, 1)), wt.float(), b, stride=2, padding=0)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, cout)
    out = ops.conv3x3_stride2(x, _prep3x3(wt), b, pad_mode=mode)
    check(f"conv3x3 stride2 {mode} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("b,t,hw,c", [(2, 17, 64, 128), (1, 9, 256, 64), (2, 5, 16, 64)])
def test_tconv3(dtype, b, t, hw, c):
    ops = _ops()
    x = _rand((b * t * hw, c), dtype, 1.0, 1)
    wt = _rand((c, c, 3, 1, 1), dtype, (3 * c) ** -0.5, 2)
    bias = _rand((c,), torch.float32, 1.0, 3)
    res = _rand((b * t * hw, c), dtype, 1.0, 4)
    x5 = x.float().reshape(b, t, hw, 1, c).permute(0, 4, 1, 2, 3)          # b c t hw 1
    ref = F.conv3d(x5, wt.float(), bias, padding=(1, 0, 0)).permute(0, 2, 3, 4, 1).reshape(-1, c) + res.float()
    wp = wt.reshape(c, c, 3).permute(0, 2, 1).reshape(c, 3 * c).contiguous()
    out = ops.tconv3(x, b, t, hw, wp, bias, residual=res)
    check(f"tconv3 b{b} t{t} hw{hw} c{c} {dtype}", out, ref, *TOL[dtype])


def test_small_cin_conv_via_padding():
    """conv_in path: 5 input channels zero-padded to 8 (inner TMA box wider than the tensor extent)."""
    ops = _ops()
    dtype = torch.float16
    nb, h, w, cout = 3, 16, 16, 64
    x5 = _rand((nb, h, w, 5), dtype, 1.0, 1)
    x8 = torch.zeros((nb, h, w, 8), device="cuda", dtype=dtype)
    x8[..., :5] = x5
    wt = _conv_weight(cout, 5, dtype, 2)
    w8 = torch.zeros((cout, 8, 3, 3), device="cuda", dtype=dtype)
    w8[:, :5] = wt
    b = _rand((cout,), torch.float32, 1.0, 3)
    ref = F.conv2d(x5.float().permute(0, 3, 1, 2), wt.float(), b, padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
    out = ops.conv3x3(x8, _prep3x3(w8), b)
    check("conv3x3 cin=5 padded to 8", out, ref, *TOL[dtype])


def test_batched_gemm_qk():
    """S = Q K^T per frame with B batched along a pixel dim (VAE mid-block attention path)."""
    ops = _ops()
    dtype = torch.float16
    f, l, d = 3, 256, 128
    qkv = _rand((f * l, 3 * d), dtype, 1.0, 1)
    q = qkv[:, :d]
    k = qkv[:, d:2 * d]
    ref = torch.einsum("fld,fmd->flm", q.float().reshape(f, l, d), k.float().reshape(f, l, d)).reshape(f * l, l) * 0.1
    out = ops.igemm(q, (d, l, f, 1, 1), (1, 3 * d, l * 3 * d, 0, 0), k, l, d, (l, f, 1, 1), (128, 1, 1, 1),
                    [[0, 0, 0, 0, 0]], ld_b=3 * d, b_batch=f, b_batch_stride=l * 3 * d, b_batch_dim=1, out_f32=True,
                    out_scale=0.1)
    check("batched QK^T", out, ref, 1e-3, 1e-3)


# ------------------------------------------------------------------------------------------------ 256-column tiles
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("m,k,n", [(256, 64, 256), (4096, 512, 512), (1000, 640, 1280), (139264 // 8, 320, 320),
                                   (384, 1280, 2560), (130, 320, 256), (8704, 1280, 1280), (640, 320, 576), (896, 2880, 320)])
def test_linear_block_n256(dtype, residual, m, k, n):
    """256-column tiles (narrowed by `fit_block_n` where N is wider than one tile): even / odd numbers of m-tiles
    (130 rows = 2 tiles, 1000 = 8, 384 = 3), ragged last n-tile (320 = 256 + 64), partial last m-tile."""
    ops = _ops()
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    ref = x.float() @ w.float().t() + b
    if residual:
        res = _rand((m, n), dtype, 1.0, 4)
        out = ops.linear(x, w, b, residual=res, block_n=256)
        check(f"linear+res bn256 {m}x{k}x{n} {dtype}", out, ref + res.float(), *TOL[dtype])
    else:
        out = ops.linear(x, w, b, block_n=256)
        check(f"linear bn256 {m}x{k}x{n} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_epilogues_block_n256(dtype):
    ops = _ops()
    # GEGLU (values | gates: two slices of the weight tile)
    m, k, n = 1500, 320, 2560
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 0.5, 3)
    y = x.float() @ w.float().t() + b
    ref = y[:, : n // 2] * F.gelu(y[:, n // 2:])
    out = ops.linear(x, w, b, geglu=True)
    check("geglu", out, ref, *TOL[dtype])
    # per-sample bias (time embedding) and SiLU epilogues
    n2 = 640
    w2 = _rand((n2, k), dtype, k ** -0.5, 4)
    b2 = _rand((3, n2), torch.float32, 1.0, 5)
    ref2 = x.float() @ w2.float().t() + b2.repeat_interleave(500, dim=0)
    check("bias2", ops.linear(x, w2, None, bias2=b2, rows_per_bias2=500, block_n=256), ref2, *TOL[dtype])
    check("silu", ops.linear(x, w2, None, act=ops.ACT_SILU, block_n=256), F.silu(x.float() @ w2.float().t()), *TOL[dtype])
    # conv 3x3 with a virtual channel concat (two-source K loop) and an odd number of m-tiles (3 x 24 x 16 px = 9 tiles)
    xa = _rand((3, 24, 16, 128), dtype, 1.0, 6)
    xb = _rand((3, 24, 16, 64), dtype, 1.0, 7)
    wc = _rand((256, 192, 3, 3), dtype, (192 * 9) ** -0.5, 8)
    wk = wc.permute(0, 2, 3, 1).reshape(256, -1).contiguous()
    refc = F.conv2d(torch.cat([xa, xb], dim=-1).permute(0, 3, 1, 2).float(), wc.float(), padding=1)
    outc = ops.conv3x3(xa, wk, None, x2=xb, block_n=256)
    check("conv3x3 concat", outc, refc.permute(0, 2, 3, 1).reshape(-1, 256), *TOL[dtype])
    # temporal 3-tap conv
    xt = _rand((2 * 5 * 64, 256), dtype, 1.0, 9)
    wt = _rand((256, 3 * 256), dtype, (3 * 256) ** -0.5, 10)
    outt = ops.tconv3(xt, 2, 5, 64, wt, None, block_n=256)
    x5 = xt.float().reshape(2, 5, 64, 256).permute(0, 3, 1, 2).unsqueeze(-1)           # b c t hw 1
    w5 = wt.float().reshape(256, 3, 256).permute(0, 2, 1).reshape(256, 256, 3, 1, 1)
    reft = F.conv3d(x5, w5, padding=(1, 0, 0)).squeeze(-1).permute(0, 2, 3, 1).reshape(-1, 256)
    check("tconv3", outt, reft, *TOL[dtype])
