"""GPU: the SVD-loop and boundary kernels against their stated contracts, written as plain torch on the same device.

Copies and permutations must match bit for bit.  Kernels that claim torch's 16-bit roundings must equal the torch op sequence
bit for bit.  Kernels with fp32 arithmetic are checked against float64 within one rounding of the 16-bit output."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, dtype, seed, scale=1.0):
    return (torch.randn(shape, device="cuda", generator=_gen(seed)) * scale).to(dtype)


def _ulp(ref64, dtype):
    """Spacing of `dtype` at |ref64| (the size of one rounding of the output)."""
    fi = torch.finfo(dtype)
    mant = {torch.float16: 10, torch.bfloat16: 7}[dtype]
    e = torch.floor(torch.log2(ref64.abs().clamp_min(fi.tiny)))
    return torch.exp2(e.clamp_min(math.log2(fi.tiny)) - mant)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------- copies and permutations
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", [9, 16, 1])
def test_image_to_nhwc16(dtype, c):
    """[N, C, H, W] with arbitrary strides -> channels-last [N, H, W, 16], channels >= C zero."""
    from animate_anything_b200 import ops
    n, h, w = 3, 5, 7
    base = _randn((n, h, c + 3, w + 4), dtype, c)
    img = base[:, :, 2:2 + c, 1:1 + w].permute(0, 2, 1, 3)                    # strided in every dimension
    out = ops.image_to_nhwc16(img)
    torch.cuda.synchronize()
    assert torch.equal(out, F.pad(img.permute(0, 2, 3, 1), (0, 16 - c)))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("ldc", [4, 16, 20])
def test_svd_out_finalize(dtype, ldc):
    """conv_out rows [(b f h w), ldc] fp32 -> [B, F, 4, H, W] 16-bit: channels 0..3 only, one rounding."""
    from animate_anything_b200 import ops
    b, f, h, w = 2, 3, 5, 6
    y = torch.randn((b * f * h * w, ldc), device="cuda", generator=_gen(ldc)) * 3
    out = ops.svd_out_finalize(y, b, f, h, w, dtype)
    torch.cuda.synchronize()
    assert torch.equal(out, y[:, :4].reshape(b, f, h, w, 4).permute(0, 1, 4, 2, 3).to(dtype))


def _unet_upsample_pairs(lo=9, hi=33, levels=4):
    """(input, output_size) of every UNet Upsample2D at latent sizes lo..hi: down with (s + 1) // 2, up back to the skip size."""
    pairs = set()
    for s in range(lo, hi + 1):
        sizes = [s]
        for _ in range(levels - 1):
            sizes.append((sizes[-1] + 1) // 2)
        pairs.update((sizes[i + 1], sizes[i]) for i in range(levels - 1))
    return sorted(pairs)


def _upsample_ref(x, oh, ow):
    return F.interpolate(x.permute(0, 3, 1, 2), size=(oh, ow), mode="nearest").permute(0, 2, 3, 1)


@pytest.mark.parametrize("dtype", DTYPES)
def test_upsample_nearest_unet_sizes(dtype):
    """Every (H -> OH) the UNet produces for latent sizes 9..33, in H and (paired with a different pair) in W."""
    from animate_anything_b200 import ops
    pairs = _unet_upsample_pairs()
    assert (5, 9) in pairs and (17, 33) in pairs and (2, 3) in pairs
    for i, (h, oh) in enumerate(pairs):
        w, ow = pairs[(i * 7 + 3) % len(pairs)]
        x = _randn((2, h, w, 8), dtype, i)
        y = ops.upsample_nearest(x, oh, ow)
        assert torch.equal(y, _upsample_ref(x, oh, ow)), ((h, oh), (w, ow))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", [8, 1280])
def test_upsample_nearest_sweep(dtype, c):
    """H in 1..17 with OH in H..2H+1, along each axis in turn."""
    from animate_anything_b200 import ops
    for h in range(1, 18):
        for oh in range(h, 2 * h + 2):
            x = _randn((1, h, 3, c), dtype, 100 * h + oh)
            assert torch.equal(ops.upsample_nearest(x, oh, 5), _upsample_ref(x, oh, 5)), (h, oh)
            xt = x.transpose(1, 2).contiguous()
            assert torch.equal(ops.upsample_nearest(xt, 5, oh), _upsample_ref(xt, 5, oh)), (h, oh)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("h,w,c", [(15, 17, 8), (9, 9, 320), (1, 1, 8), (16, 17, 64), (17, 16, 64), (3, 33, 1280)])
def test_pad_to_even(dtype, h, w, c):
    from animate_anything_b200 import ops
    x = _randn((2, h, w, c), dtype, h * w)
    y = ops.pad_to_even(x)
    assert torch.equal(y, F.pad(x, (0, 0, 0, w & 1, 0, h & 1)))
    if h % 2 == 0 and w % 2 == 0:
        assert y is x


@pytest.mark.parametrize("dtype", DTYPES)
def test_dup_rows(dtype):
    """Both halves equal the input, and the producer's column statistics travel with the rows."""
    from animate_anything_b200 import ops
    x = _randn((256, 40), dtype, 3)
    stats = torch.randn((2, 40, 2), device="cuda", generator=_gen(4))
    x._aab_stats = stats
    out = ops.dup_rows(x)
    torch.cuda.synchronize()
    assert torch.equal(out, torch.cat([x, x]))
    assert torch.equal(out._aab_stats, torch.cat([stats, stats]))
    odd = _randn((3, 8), dtype, 5)                                  # 48 bytes: three 16-byte units
    assert torch.equal(ops.dup_rows(odd), torch.cat([odd, odd]))


@pytest.mark.parametrize("dtype", DTYPES)
def test_copy2d_both_paths(dtype):
    """`cat_cols` with an odd first width (second copy misaligned -> scalar path), and `aab_copy2d` on both of its paths
    into a sentinel-filled destination: the block is copied and nothing outside it is written."""
    from animate_anything_b200 import _lib, ops
    x = _randn((77, 13), dtype, 1)
    x2 = _randn((77, 24), dtype, 2)
    assert torch.equal(ops.cat_cols(x, x2), torch.cat([x, x2], dim=1))
    wide = _randn((77, 40), dtype, 3)
    assert torch.equal(ops.cat_cols(wide[:, 3:17], wide[:, 1:9]), torch.cat([wide[:, 3:17], wide[:, 1:9]], dim=1))
    src = _randn((50, 48), dtype, 4)
    # (misaligned bases: scalar), (odd width: scalar), (16-byte aligned: vector), (vector)
    for (r0, c0, rows, cols, dc0) in [(1, 3, 20, 11, 5), (0, 0, 10, 13, 0), (0, 8, 33, 24, 16), (2, 0, 48, 16, 8)]:
        dst = torch.full((60, 48), -7.0, device="cuda", dtype=dtype)
        want = dst.clone()
        want[r0:r0 + rows, dc0:dc0 + cols] = src[r0:r0 + rows, c0:c0 + cols]
        s = src[r0:, c0:]
        d = dst[r0:, dc0:]
        _lib.call("aab_copy2d", C.c_void_p(s.data_ptr()), src.stride(0), C.c_void_p(d.data_ptr()), dst.stride(0), rows, cols,
                  _stream())
        torch.cuda.synchronize()
        assert torch.equal(dst, want), (r0, c0, rows, cols, dc0)


@pytest.mark.parametrize("dtype", DTYPES)
def test_embed_tokens(dtype):
    """tok[ids] + pos[r % L] with torch's 16-bit add; ids at 0 and vocab - 1; a partial last sequence."""
    from animate_anything_b200 import ops
    vocab, c, seq = 1000, 64, 7
    tok = _randn((vocab, c), dtype, 1)
    pos = _randn((seq, c), dtype, 2)
    for rows in (3 * seq, 2 * seq + 3, 1):
        ids = torch.randint(0, vocab, (rows,), device="cuda", generator=_gen(rows))
        ids[0] = 0
        ids[-1] = vocab - 1
        out = ops.embed_tokens(ids, tok, pos, seq)
        torch.cuda.synchronize()
        assert torch.equal(out, tok[ids] + pos[torch.arange(rows, device="cuda") % seq]), rows


# ---------------------------------------------------------------------------------------------- add_rowvec
def _rowvec_index(rows, rows_per_vec, mod, mode, mod2):
    """Index of the vector each row reads, from the documented meaning rather than the kernel's formula."""
    if mode == 0:                                    # row block r // rows_per_vec, cycling over `mod` vectors
        return torch.tensor([(r // rows_per_vec) % mod for r in range(rows)])
    s_len, f_len = rows_per_vec, mod2                # rows (b, f, s): token (b, s) of every frame reads (b * S + s) % mod
    idx = []
    for b in range(rows // (s_len * f_len)):
        for _f in range(f_len):
            idx.extend((b * s_len + s) % mod for s in range(s_len))
    return torch.tensor(idx)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode,b,f,s,mod", [(1, 1, 3, 5, 1), (1, 2, 3, 5, 2), (1, 3, 4, 7, 3), (1, 2, 3, 5, 3), (1, 3, 2, 4, 5),
                                            (0, 2, 3, 5, 2), (0, 3, 4, 7, 4), (0, 1, 1, 9, 1)])
@pytest.mark.parametrize("inplace", [False, True])
def test_add_rowvec(dtype, mode, b, f, s, mod, inplace):
    """out = x + vec[idx(r)] in fp32, rounded once; x and vec with row strides wider than `cols`; in place through a
    strided x.  Mode 0 is exercised with rows_per_vec = S (per-frame vectors, mod = F) or F*S (per-sample, mod = B)."""
    from animate_anything_b200 import ops
    cols = 40
    rows = b * f * s
    if mode == 0:
        rows_per_vec, mod2 = (s, 1) if mod == f else (f * s, 1)
    else:
        rows_per_vec, mod2 = s, f
    nvec = max(mod, 1)
    xbuf = _randn((rows, cols + 16), dtype, rows, 2.0)
    x = xbuf[:, 8:8 + cols]
    vbuf = torch.randn((nvec, cols + 12), device="cuda", generator=_gen(7)) * 3
    vec = vbuf[:, :cols]
    idx = _rowvec_index(rows, rows_per_vec, mod, mode, mod2).cuda()
    assert idx.numel() == rows
    exact = (x.float() + vec[idx]).to(dtype)                          # fp32 add, one rounding
    ref64 = x.double() + vec.double()[idx]
    before = xbuf.clone()
    out = ops.add_rowvec(x, vec, rows_per_vec, mod, mode=mode, mod2=mod2, inplace=inplace)
    torch.cuda.synchronize()
    assert torch.equal(out, exact)
    assert bool(((out.double() - ref64).abs() <= _ulp(ref64, dtype)).all())
    if inplace:
        assert out.data_ptr() == x.data_ptr()
        assert torch.equal(xbuf[:, :8], before[:, :8]) and torch.equal(xbuf[:, 8 + cols:], before[:, 8 + cols:])
    else:
        assert torch.equal(xbuf, before)


# ---------------------------------------------------------------------------------------------- axpby (AlphaBlender)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("coef", ["alpha0.5", "alpha-0.37", "alpha1.3", "free"])
def test_axpby(dtype, coef):
    """a * x + b * y with Python-float a, b on 16-bit CUDA tensors, bit for bit: the product and sum roundings of torch with
    fp32 coefficients.  The AlphaBlender coefficients are sigmoid(mix_factor) in fp32 and 1 - that (not rounded to dtype)."""
    from animate_anything_b200 import ops
    if coef == "free":
        a, b = 0.3, -1.7
    else:
        a = float(torch.sigmoid(torch.tensor(float(coef[5:]))).item())
        b = 1.0 - a
    n = 64 * 1031
    x = _randn((n,), dtype, 1) * _randn((n,), dtype, 2).abs().exp()        # magnitudes over several binades
    y = _randn((n,), dtype, 3) * 4
    out = ops.axpby(x, y, a, b)
    torch.cuda.synchronize()
    assert torch.equal(out, a * x + b * y)


# ---------------------------------------------------------------------------------------------- SVD loop boundary
def _svd_sigmas(steps=5):
    from oracle.composition import SVD_SCHED
    from animate_anything_b200.schedulers import EulerDiscreteScheduler
    s = EulerDiscreteScheduler(**SVD_SCHED)
    s.set_timesteps(steps)
    sig = [float(v) for v in s.sigmas]
    assert sig[-1] == 0.0 and sig[0] > 100
    return sig


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,f", [(1, 1), (2, 14), (2, 1), (1, 14)])
@pytest.mark.parametrize("cfg", [True, False])
def test_svd_in_assemble(dtype, b, f, cfg):
    """[(2)B*F, h, w, 16]: channel 0 the [h, w] mask broadcast to every (b, f); 1..4 x * fp32(1/sqrt(sigma^2+1)) rounded once;
    5..8 the image latent of sample b for every frame, zeros in the unconditional (first) half; 9..15 zero."""
    from animate_anything_b200 import ops
    h, w = 5, 7
    x = _randn((b, f, 4, h, w), dtype, 1, 80.0)
    img = _randn((b, 4, h, w), dtype, 2)
    mask = _randn((h, w), dtype, 3)
    for sigma in _svd_sigmas()[:-1:2]:
        out = ops.svd_in_assemble(x, img, mask, sigma, cfg)
        torch.cuda.synchronize()
        inv = float(torch.tensor(1.0 / math.sqrt(sigma * sigma + 1.0), dtype=torch.float32))
        xs = (x.float() * inv).to(dtype)
        halves = []
        for cond in ((False, True) if cfg else (True,)):
            lat = img if cond else torch.zeros_like(img)
            ch = torch.cat([mask.expand(b, f, 1, h, w), xs, lat[:, None].expand(b, f, 4, h, w),
                            torch.zeros((b, f, 7, h, w), device="cuda", dtype=dtype)], dim=2)
            halves.append(ch.reshape(b * f, 16, h, w).permute(0, 2, 3, 1))
        assert torch.equal(out, torch.cat(halves)), sigma


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,f", [(1, 1), (2, 14), (1, 14)])
@pytest.mark.parametrize("cfg", [True, False])
def test_svd_cfg_euler_step(dtype, b, f, cfg):
    """Guidance with torch's 16-bit roundings (bit for bit against the torch op sequence), then the v-prediction Euler step in
    fp32 (float64 reference: within one rounding of the output, and nearly always the correctly rounded value -- which a
    16-bit rounding of v * (-sigma / sqrt(sigma^2 + 1)) would break for about a quarter of the outputs at the middle
    step, sigma ~ 0.68).  pred is a conv_out-like
    [rows, 16] fp32 matrix; gs = linspace(1, 3, F) unrounded; the real SVD sigmas including the last step to 0."""
    from animate_anything_b200 import ops
    h, w = 6, 5
    nb = 2 * b if cfg else b
    pred = torch.randn((nb * f * h * w, 16), device="cuda", generator=_gen(1))
    pred[:, 4:] = 1e4                                                    # channels the kernel must not read
    gs = torch.linspace(1.0, 3.0, f, device="cuda")
    sig = _svd_sigmas()
    for i in (0, len(sig) // 2, len(sig) - 2):
        sigma, sigma_next = sig[i], sig[i + 1]
        x = _randn((b, f, 4, h, w), dtype, 10 + i, max(1.0, sigma * 0.5))
        out = ops.svd_cfg_euler_step(pred, cfg, gs if cfg else None, x, sigma, sigma_next)
        torch.cuda.synchronize()
        p16 = pred[:, :4].to(dtype).reshape(nb, f, h, w, 4).permute(0, 1, 4, 2, 3)
        if cfg:
            g16 = gs.to(dtype).reshape(1, f, 1, 1, 1)
            v = p16[:b] + g16 * (p16[b:] - p16[:b])                     # 16-bit tensor ops, as diffusers on fp16 latents
        else:
            v = p16
        s = float(torch.tensor(sigma, dtype=torch.float32))
        sn = float(torch.tensor(sigma_next, dtype=torch.float32))
        xs = x.double()
        x0 = v.double() * (-s / math.sqrt(s * s + 1.0)) + xs / (s * s + 1.0)
        ref = xs + (xs - x0) / s * (sn - s)
        err = (out.double() - ref).abs()
        # one rounding of the output, plus the fp32 evaluation error of terms as large as x (cancellation in x - x0)
        tol = _ulp(ref, dtype) + 2.0 ** -20 * (xs.abs() + v.double().abs())
        assert bool((err <= tol).all()), (i, float((err - tol).max()))
        mismatch = (out != ref.to(dtype)).double().mean().item()
        assert mismatch <= 0.02, (i, mismatch)


# ---------------------------------------------------------------------------------------------- cast_f32
def _ties_and_neighbours(dtype, n, seed):
    """fp32 values halfway between consecutive finite `dtype` values, and one fp32 ulp either side of them."""
    g = torch.Generator().manual_seed(seed)
    bits = torch.randint(0, 0x7BFF if dtype == torch.float16 else 0x7F7F, (n,), generator=g, dtype=torch.int32)
    lo = bits.to(torch.int16).view(dtype).float()
    hi = (bits + 1).to(torch.int16).view(dtype).float()
    mid = (lo.double() + hi.double()) / 2
    mid32 = mid.float()
    assert torch.equal(mid32.double(), mid)                       # exactly representable in fp32
    sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    up = torch.nextafter(mid32, torch.full_like(mid32, math.inf))
    dn = torch.nextafter(mid32, torch.full_like(mid32, -math.inf))
    return torch.cat([mid32, up, dn, lo]) * sign.repeat(4)


@pytest.mark.parametrize("dtype", DTYPES)
def test_cast_f32_special_values(dtype):
    """`aab_cast_f32` against `.to(dtype)`: +-inf, NaN, the largest finite value and its fp32 neighbours, values that
    overflow, subnormals of both formats, and round-to-nearest-even ties."""
    from animate_anything_b200 import _lib
    inf = math.inf
    fmax = torch.finfo(dtype).max
    top = torch.tensor([fmax], dtype=torch.float32)
    special = [inf, -inf, math.nan, 0.0, -0.0, fmax, -fmax, torch.finfo(torch.float32).max, -torch.finfo(torch.float32).max,
               float(torch.nextafter(top, top * 2)), float(torch.nextafter(top, top * 0)),
               torch.finfo(dtype).tiny, torch.finfo(dtype).tiny / 2, torch.finfo(torch.float32).tiny,
               torch.finfo(torch.float32).tiny / 3, 1.401298464324817e-45]
    if dtype == torch.float16:
        special += [65519.99609375, 65520.0, -65520.0, 2.0 ** -24, 2.0 ** -25, 1.5 * 2.0 ** -25, 3.0 * 2.0 ** -26]
    else:
        special += [float(torch.tensor(fmax, dtype=torch.float64) * (1 + 2.0 ** -8))]
    g = torch.Generator().manual_seed(0)
    sub = torch.randint(1, 1 << 23, (4096,), generator=g, dtype=torch.int32).view(torch.float32)   # fp32 subnormals
    small = torch.rand(4096, generator=g) * 2.0 ** -13                                                # fp16 subnormal range
    x = torch.cat([torch.tensor(special, dtype=torch.float32), sub, -sub, small, -small,
                   _ties_and_neighbours(dtype, 20000, 1), torch.randn(20000, generator=g) * 1e3]).cuda()
    y = torch.empty(x.shape, device="cuda", dtype=dtype)
    _lib.call("aab_cast_f32", C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), x.numel(), int(dtype == torch.bfloat16),
              _stream())
    torch.cuda.synchronize()
    want = x.to(dtype)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(y), nan)
    assert torch.equal(y[~nan].view(torch.int16), want[~nan].view(torch.int16))        # bits: signed zeros, infinities


# ---------------------------------------------------------------------------------------------- VAE boundary
def _finite_16bit_values(dtype):
    """Every finite value of `dtype`, as float32."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    v = bits.view(dtype).float()
    return v[torch.isfinite(v)]


def _dec_rows(values, b, f, h, w, ldc, seed):
    """conv_out-like rows [b*f*h*w, ldc] fp32 carrying `values` (cycled) in channels 0..2; the other channels hold values
    the kernels must not read."""
    n = b * f * h * w
    assert 3 * n >= values.numel()
    perm = torch.randperm(3 * n, generator=torch.Generator().manual_seed(seed)) % values.numel()
    y = torch.full((n, ldc), 1e4)
    y[:, :3] = values[perm].reshape(n, 3)
    return y.cuda()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rint", [False, True])
def test_vae_dec_finalize_u8_every_value(dtype, rint):
    """Every finite 16-bit value through both roundings, B = 2 and ldc = 5, into the [f, h, b*w, 3] frames.  The kernel
    depends only on the 16-bit rounding of its input, so this is exhaustive.  The reference is the op sequence of
    diffusers: tensor2vid `video.mul_(0.5).add_(0.5).clamp_(0, 1)` then numpy `(x * 255).astype("uint8")` (truncation);
    `postprocess(output_type="pil")`: `(x / 2 + 0.5).clamp(0, 1)`, numpy `(x * 255).round().astype("uint8")`.
    +-inf, and fp32 inputs of +-1e6 and +-3e38 (+-inf after an fp16 rounding), give 255 and 0: the clamp saturates them."""
    from animate_anything_b200 import ops
    import numpy as np
    b, f, h, w, ldc = 2, 4, 64, 48, 5
    vals = _finite_16bit_values(dtype)
    y = _dec_rows(vals, b, f, h, w, ldc, 1)
    y[:6, 0] = torch.tensor([math.inf, -math.inf, 1e6, -1e6, 3e38, -3e38], device="cuda")
    out = ops.vae_dec_finalize_u8(y, b, f, h, w, dtype == torch.bfloat16, round_half_even=rint)
    torch.cuda.synchronize()
    video = y[:, :3].to(dtype).float().reshape(b, f, h, w, 3).permute(0, 4, 1, 2, 3)          # decode_latents output
    if rint:
        x = ((video / 2 + 0.5).clamp(0, 1)).permute(2, 3, 0, 4, 1).reshape(f, h, b * w, 3).cpu().numpy()
        want = (x * np.float32(255)).round().astype("uint8")
    else:
        x = video.mul(0.5).add(0.5).clamp(0, 1).permute(2, 3, 0, 4, 1).reshape(f, h, b * w, 3).cpu().numpy()
        want = (x * np.float32(255)).astype("uint8")
    assert x.dtype == np.float32
    assert torch.equal(out.cpu(), torch.from_numpy(want))
    # pixel (b=0, f=0, y=0, x=0..5) channel 0: +inf, -inf, and the 16-bit overflows
    assert out[0, 0, :6, 0].tolist() == [255, 0, 255, 0, 255, 0]


@pytest.mark.parametrize("dtype", DTYPES)
def test_vae_dec_finalize_every_value(dtype):
    """conv_out rows -> float32 video [B, 3, F, H, W]: every finite 16-bit value, plus round-to-nearest-even ties and their
    fp32 neighbours, rounded once to the model dtype, bit for bit."""
    from animate_anything_b200 import ops
    b, f, h, w, ldc = 2, 4, 64, 48, 5
    vals = torch.cat([_finite_16bit_values(dtype), _ties_and_neighbours(dtype, 2000, 3)])
    y = _dec_rows(vals, b, f, h, w, ldc, 2)
    out = ops.vae_dec_finalize(y, b, f, h, w, dtype == torch.bfloat16)
    torch.cuda.synchronize()
    want = y[:, :3].to(dtype).float().reshape(b, f, h, w, 3).permute(0, 4, 1, 2, 3)
    assert torch.equal(out.view(torch.int32), want.contiguous().view(torch.int32))


@pytest.mark.parametrize("dtype", DTYPES)
def test_vae_enc_finalize_scaled(dtype):
    """quant_conv then the 0.18215 latent scale, ldm = 16: the reference rounds the moments to the model dtype and then
    multiplies the 16-bit tensor (two roundings).  Against float64: within one output ulp plus the half ulp of the
    intermediate rounding, scaled (and 2^-20 of sum |w m| for the fp32 accumulation).  The double rounding itself:
    the torch sequence round16(round16(acc) * scale) is matched except where fp32 and float64 accumulation straddle an
    intermediate rounding boundary, while a single rounding of acc * scale differs for a sizeable share of the outputs."""
    from animate_anything_b200 import ops
    b, f, h, w, ldm, scale = 2, 3, 8, 12, 16, 0.18215
    mom = _randn((b * f * h * w, ldm), dtype, 1, 3.0)
    wq = torch.randn((8, 8), device="cuda", generator=_gen(2)) * 0.5
    bq = torch.randn((8,), device="cuda", generator=_gen(3)) * 0.5
    out = ops.vae_enc_finalize(mom, wq, bq, scale, b, f, h, w)
    torch.cuda.synchronize()

    def layout(t):
        return t.reshape(b, f, h, w, 8).permute(0, 4, 1, 2, 3)
    m = mom[:, :8].double()
    acc = layout(m @ wq.double().t() + bq.double())
    mag = layout(m.abs() @ wq.double().abs().t() + bq.double().abs())
    ref = acc * scale
    tol = _ulp(ref, dtype) + scale * (_ulp(acc, dtype) / 2 + 2.0 ** -20 * mag)
    err = (out.double() - ref).abs()
    assert bool((err <= tol).all()), float((err / tol).max())
    s32 = float(torch.tensor(scale, dtype=torch.float32))
    double = (acc.to(dtype).float() * s32).to(dtype)
    single = (acc * s32).to(dtype)
    assert (out != double).double().mean().item() <= 0.01
    assert (double != single).double().mean().item() >= 0.05


@pytest.mark.parametrize("dtype", DTYPES)
def test_vae_dec_in(dtype):
    """latents / 0.18215 rounded to the model dtype (torch's fp32 multiply, bit for bit the same z), post_quant_conv in
    fp32 (float64 reference: one output ulp plus 2^-20 of sum |w z| + |b|), channels 4..7 exactly +0."""
    from animate_anything_b200 import ops
    b, f, h, w = 2, 3, 8, 12
    lat = _randn((b, 4, f, h, w), dtype, 5, 0.9)
    wp = torch.randn((4, 4), device="cuda", generator=_gen(6)) * 0.5
    bp = torch.randn((4,), device="cuda", generator=_gen(7)) * 0.5
    inv = 1 / 0.18215
    out = ops.vae_dec_in(lat, inv, wp, bp)
    torch.cuda.synchronize()
    assert torch.equal(out[..., 4:].view(torch.int16), torch.zeros_like(out[..., 4:]).view(torch.int16))
    z = (lat.float() * float(torch.tensor(inv, dtype=torch.float32))).to(dtype).double()
    z = z.permute(0, 2, 3, 4, 1).reshape(-1, 4)
    ref = z @ wp.double().t() + bp.double()
    tol = _ulp(ref, dtype) + 2.0 ** -20 * (z.abs() @ wp.double().abs().t() + bp.double().abs())
    err = (out.reshape(-1, 8)[:, :4].double() - ref).abs()
    assert bool((err <= tol).all()), float((err / tol).max())


# ---------------------------------------------------------------------------------------------- UNet loop boundary
def _get_timestep_embedding(t, dim):
    """diffusers embeddings.get_timestep_embedding(t, dim, flip_sin_to_cos=True, downscale_freq_shift=0), fp32."""
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    return torch.cat([emb[:, half:], emb[:, :half]], dim=-1)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dim", [256, 320, 1280])
def test_timestep_embed(dtype, dim):
    """t_count in {1, B/2 (CFG: [uncond..., text...]), B}; t = 0, 1, 999 and the SVD noise-level inputs 0.25 * log(sigma).
    Against diffusers' fp32 embedding: one ulp of the model dtype plus 2^-21 |t * freq|.  Two fp32 evaluations of the
    argument t * freq differ by up to ~4 of its fp32 roundings (expf is within 2 ulp, and the product rounds once more),
    and sin / cos pass that on unchanged: at t = 999 that is ~2.4e-4, several fp16 ulps of a small output, so "one ulp"
    alone holds only for the small t.  float64 sanity bound: one ulp plus 2^-20 (|t * freq| + 1), the same argument error
    and that of sinf / cosf."""
    from animate_anything_b200 import ops
    b = 8
    vals = [0.0, 1.0, 999.0] + [0.25 * math.log(s) for s in _svd_sigmas()[:-1]]
    assert len(vals) == b and any(v != int(v) for v in vals)
    half = dim // 2
    freq64 = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float64, device="cuda") / half)
    for tc in (1, b // 2, b):
        for start in range(0, b, tc):
            t = torch.tensor(vals[start:start + tc], device="cuda", dtype=torch.float32)
            out = ops.timestep_embed(t, b, dim, dtype)
            torch.cuda.synchronize()
            tb = t.repeat(b // tc)                                      # row r takes t[r % t_count]
            ref32 = _get_timestep_embedding(tb, dim)
            arg = tb.double()[:, None] * freq64[None]
            arg2 = torch.cat([arg, arg], -1).abs()
            err = (out.double() - ref32.double()).abs()
            tol = _ulp(ref32.double(), dtype) + 2.0 ** -21 * arg2
            assert bool((err <= tol).all()), (tc, start, float((err / tol).max()))
            if float(tb.abs().max()) <= 2:
                assert bool((err <= _ulp(ref32.double(), dtype)).all()), (tc, start)
            ref64 = torch.cat([torch.cos(arg), torch.sin(arg)], -1)
            tol = _ulp(ref64, dtype) + 2.0 ** -20 * (arg2 + 1)
            assert bool(((out.double() - ref64).abs() <= tol).all()), (tc, start)


def _coef_rows(kind, steps=10):
    from animate_anything_b200.schedulers import DDIMScheduler, DPMSolverMultistepScheduler
    common = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    if kind == "ddim":
        s = DDIMScheduler(clip_sample=False, set_alpha_to_one=False, steps_offset=1, **common)
    else:
        s = DPMSolverMultistepScheduler(**common)
    s.set_timesteps(steps)
    table, hist = s.step_coefficients(s.timesteps)
    return torch.from_numpy(table).cuda(), hist


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["ddim", "dpm"])
@pytest.mark.parametrize("cfg", [True, False])
def test_cfg_scheduler_step_coefficients(dtype, kind, cfg):
    """n = 2 prompts (CFG pairs sample b with b + n), the real DDIM / DPM-Solver++ coefficient tables at step 5, with the
    x0 history (DPM-Solver++) and without (DDIM passes None).  float64 reference: one output ulp plus 2^-20 of the sum of
    the magnitudes of the fp32 terms; the history within 2^-20 of its terms."""
    from animate_anything_b200 import ops
    n, f, h, w, ldc, g = 2, 3, 6, 5, 16, 7.5
    t = f + 1
    nb = 2 * n if cfg else n
    coef, needs_hist = _coef_rows(kind)
    assert needs_hist == (kind == "dpm")
    step = torch.tensor([5], device="cuda", dtype=torch.int32)
    eps = torch.randn((nb * t * h * w, ldc), device="cuda", generator=_gen(1))
    eps[:, 4:] = 1e4                                                   # channels the kernel must not read
    x = _randn((n, 4, f, h, w), dtype, 2, 2.0)
    hist = torch.randn((n, 4, f, h, w), device="cuda", generator=_gen(3)) if needs_hist else None
    hist0 = hist.clone() if needs_hist else None
    out = torch.empty_like(x)
    ops.cfg_scheduler_step(eps, ldc, cfg, g, x, out, hist, coef, step)
    torch.cuda.synchronize()
    e4 = eps.double().reshape(nb, t, h, w, ldc)[..., :4].permute(0, 4, 1, 2, 3)[:, :, 1:]
    if cfg:
        e = e4[:n] + g * (e4[n:] - e4[:n])
        emag = e4[:n].abs() + g * (e4[n:].abs() + e4[:n].abs())
    else:
        e, emag = e4, e4.abs()
    k = coef[5].double()
    xd = x.double()
    x0 = k[0] * xd + k[1] * e
    x0mag = (k[0] * xd).abs() + k[1].abs() * emag
    ref = k[2] * xd + k[3] * e + k[4] * x0
    mag = (k[2] * xd).abs() + k[3].abs() * emag + k[4].abs() * x0mag
    if needs_hist:
        ref = ref + k[5] * hist0.double()
        mag = mag + (k[5] * hist0.double()).abs()
        assert bool(((hist.double() - x0).abs() <= 2.0 ** -20 * x0mag).all())
    err = (out.double() - ref).abs()
    tol = _ulp(ref, dtype) + 2.0 ** -20 * mag
    assert bool((err <= tol).all()), float((err / tol).max())


@pytest.mark.parametrize("dtype", DTYPES)
def test_unet_in_assemble_per_sample_masks(dtype):
    """mask_batch = B with a different mask per sample; sample, cond and mask are non-contiguous views; bit for bit."""
    from animate_anything_b200 import ops
    b, f, h, w = 3, 4, 6, 10
    sample = _randn((b, f, h, w, 4), dtype, 1).permute(0, 4, 1, 2, 3)            # channels-last storage
    cond = _randn((b, 4, 3, h, w + 2), dtype, 2)[:, :, 1:2, :, 1:1 + w]
    mask = (_randn((b, 2, 1, h, w), dtype, 3) > 0).to(dtype)[:, 1:]
    assert not (sample.is_contiguous() or cond.is_contiguous() or mask.is_contiguous())
    assert not all(torch.equal(mask[0], mask[i]) for i in range(1, b))
    out = ops.unet_in_assemble(sample, cond, mask, f + 1)
    torch.cuda.synchronize()
    ref = torch.cat([mask.expand(b, 1, f + 1, h, w), torch.cat([cond, sample], dim=2)], dim=1).permute(0, 2, 3, 4, 1)
    assert torch.equal(out[..., :5], ref.contiguous())
    assert torch.equal(out[..., 5:].view(torch.int16), torch.zeros_like(out[..., 5:]).view(torch.int16))
