"""GPU: GroupNorm (two-pass and column-statistics paths), LayerNorm, the row softmax and the VAE mid-block attention chain
against float64 references on the same 16-bit inputs.

Every comparison allows one rounding of the 16-bit output (`_ulp`) plus a slack for the kernel's fp32 arithmetic, derived
next to the assertion; copies and padding are checked bit for bit."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, dtype, seed, scale=1.0, shift=0.0):
    return (torch.randn(shape, device="cuda", generator=_gen(seed)) * scale + shift).to(dtype)


def _ulp(ref64, dtype):
    """Spacing of `dtype` at |ref64| (the size of one rounding of the output)."""
    fi = torch.finfo(dtype)
    mant = {torch.float16: 10, torch.bfloat16: 7}[dtype]
    e = torch.floor(torch.log2(ref64.abs().clamp_min(fi.tiny)))
    return torch.exp2(e.clamp_min(math.log2(fi.tiny)) - mant)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _affine(c, seed):
    gamma = (torch.randn(c, device="cuda", generator=_gen(seed)) * 0.2 + 1.0)
    beta = torch.randn(c, device="cuda", generator=_gen(seed + 1)) * 0.2
    return gamma, beta


# ---------------------------------------------------------------------------------------------- GroupNorm
def _gn_ref(x, samples, rows, groups, gamma, beta, eps, silu):
    """float64 GroupNorm (+ SiLU) of x [samples*rows, C] (any row stride), the normalised value z and the per-element
    mean/std ratio r of its group."""
    c = x.shape[1]
    xr = x.double().reshape(samples, rows, c).permute(0, 2, 1)
    pre = F.group_norm(xr, groups, gamma.double(), beta.double(), eps)
    xg = xr.reshape(samples, groups, -1)
    mean, var = xg.mean(-1, keepdim=True), xg.var(-1, unbiased=False, keepdim=True)
    z = ((xg - mean) / torch.sqrt(var + eps)).reshape(samples, c, rows)
    r = (mean.abs() / torch.sqrt(var + eps)).expand_as(xg).reshape(samples, c, rows)
    ref = F.silu(pre) if silu else pre

    def flat(t):
        return t.permute(0, 2, 1).reshape(samples * rows, c)
    return flat(ref), flat(z), flat(r)


def _gn_bound(ref, z, r, gamma, beta, silu, dtype):
    """One rounding of the output plus the fp32 error of the kernel.
    Statistics: sums of x and x^2 in fp32 chains of at most ~100 terms (per-thread row walk + per-CTA combine, or a 128-row
    tile of the producing GEMM), then fp64: E[x^2] carries a relative error d <= ~100 * 2^-24 < 2^-17 in the worst case
    (about 2^-21 for random rounding).  var = E[x^2] - mean^2 amplifies that by E[x^2] / var = 1 + r^2, and the normalised
    value z moves by half the relative error of var, plus a mean error of d * r standard deviations:
        |dz| <= 2^-18 * ((1 + r^2) * |z| + r)        -- the cancellation term, ~ r^2 * 2^-18 * |z| for large r
    Apply: fma(x, rstd * gamma, beta - mean * rstd * gamma) adds a few fp32 roundings of terms as large as
    |gamma| * (|z| + r) and |beta|.  SiLU (ex2 / rcp approximations, ~2^-21 relative) is 1.1-Lipschitz."""
    g = gamma.double().abs()
    pre = 2.0 ** -18 * (g * ((1 + r * r) * z.abs() + r + 1) + beta.double().abs())
    slack = 1.1 * pre + 2.0 ** -19 * ref.abs() if silu else pre
    return _ulp(ref, dtype) + slack


def _check_gn(y, x, samples, rows, groups, gamma, beta, eps, silu, what):
    ref, z, r = _gn_ref(x, samples, rows, groups, gamma, beta, eps, silu)
    err = (y.double() - ref).abs()
    tol = _gn_bound(ref, z, r, gamma, beta, silu, y.dtype)
    assert torch.isfinite(y).all(), what
    assert bool((err <= tol).all()), (what, float((err / tol).max()))
    return err, ref


def _rows_per_iteration(c):
    return max(1, 256 // (c // 8))


# (C, groups, eps) of every call site: UNet levels and skip concats (32 groups), VAE (eps 1e-6), UNet384 alpha decoder
# (4 groups); then one channel per group and the narrowest C
GN_SITES = [(320, 32, 1e-5), (640, 32, 1e-5), (960, 32, 1e-5), (1280, 32, 1e-5), (1920, 32, 1e-5), (2560, 32, 1e-5),
            (128, 32, 1e-6), (256, 32, 1e-6), (512, 32, 1e-6),
            (32, 4, 1e-6), (64, 4, 1e-6), (128, 4, 1e-6), (256, 4, 1e-6),
            (32, 32, 1e-5), (8, 4, 1e-5)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c,groups,eps", GN_SITES)
def test_groupnorm_call_sites(dtype, c, groups, eps):
    """Two-pass path at rows = 1, fewer than one row iteration, and a count that is not a multiple of it."""
    from animate_anything_b200 import ops
    rpi = _rows_per_iteration(c)
    gamma, beta = _affine(c, c)
    for rows in sorted({1, max(1, rpi - 1), 37 * rpi + 1}):
        for silu, samples in ((True, 2), (False, 3)):
            x = _randn((samples * rows, c), dtype, rows + c, 1.5, 0.3)
            y = ops.groupnorm(x, samples, rows, gamma, beta, eps, silu, groups)
            _check_gn(y, x, samples, rows, groups, gamma, beta, eps, silu, (c, groups, rows, silu))


def _gn_launch_cfg(c, rows):
    """Restatement of gn_launch_cfg (norm.cu): (rows per iteration, rows per CTA, chunks per sample)."""
    rpi = _rows_per_iteration(c)
    elems = rows * c
    tgt = 12288 if elems < (1 << 18) else (18432 if c >= 1280 and elems < (1 << 23) else 73728)
    rpc = max(-(-tgt // c), 8 * rpi)
    if -(-rows // rpc) > 1024:
        rpc = -(-rows // 1024)
    rpc = -(-rpc // rpi) * rpi
    return rpi, rpc, -(-rows // rpc)


@pytest.mark.parametrize("dtype", DTYPES)
def test_groupnorm_chunk_cap(dtype):
    """C = 128 over 640 x 1024 rows (a VAE decoder level-0 frame): 576 rows per CTA would give 1138 chunks, the cap raises
    it to 640 rows and exactly 1024 chunks; two samples."""
    from animate_anything_b200 import _lib, ops
    c, rows, samples, groups = 128, 640 * 1024, 2, 32
    rpi, rpc, chunks = _gn_launch_cfg(c, rows)
    assert (rpi, rpc, chunks) == (16, 640, 1024) and -(-rows // (73728 // c)) > 1024
    # the workspace size the library reports encodes its chunk count: header + mean/rstd + fp64 partials
    need = _lib.load().aab_groupnorm_workspace_bytes(samples, rows, c, groups)
    assert need == 16384 + -(-samples * groups * 8 // 256) * 256 + samples * chunks * groups * 16
    gamma, beta = _affine(c, 1)
    x = _randn((samples * rows, c), dtype, 2, 1.5, 0.3)
    y = ops.groupnorm(x, samples, rows, gamma, beta, 1e-6, True)
    _check_gn(y, x, samples, rows, groups, gamma, beta, 1e-6, True, "chunk cap")


def _producer(m, c, dtype, seed, shift=0.0):
    """A GEMM output with the column statistics of its epilogue attached (the GroupNorm column-statistics path):
    [m, 64] @ [c, 64]^T with unit-variance outputs, plus a bias `shift` (the group means)."""
    from animate_anything_b200 import ops
    x = _randn((m, 64), dtype, seed)
    w = _randn((c, 64), dtype, seed + 1, 0.125)
    bias = torch.full((c,), float(shift), device="cuda") + torch.randn(c, device="cuda", generator=_gen(seed + 2)) * 0.1
    h = ops.linear(x, w, bias, stats=True)
    assert getattr(h, "_aab_stats", None) is not None, "the producer did not emit column statistics"
    return h


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c1,c2", [(640, 320), (1280, 640)])
def test_groupnorm_concat_split_inside_a_group(dtype, c1, c2):
    """Virtual concat whose split falls inside a group (30 or 60 channels per group, split at channel 640 or 1280 =
    21 1/3 groups), through the column-statistics path and the two-pass path; strided sources for the latter."""
    from animate_anything_b200 import ops
    samples, rows = 2, 256
    gamma, beta = _affine(c1 + c2, 3)
    h1 = _producer(samples * rows, c1, dtype, 10)
    h2 = _producer(samples * rows, c2, dtype, 20, shift=-0.7)
    xc = torch.cat([h1, h2], 1)
    y = ops.groupnorm(h1, samples, rows, gamma, beta, 1e-5, True, x2=h2)
    _check_gn(y, xc, samples, rows, 32, gamma, beta, 1e-5, True, "colstats concat")
    w1 = torch.zeros((samples * rows, c1 + 24), device="cuda", dtype=dtype)
    w2 = torch.zeros((samples * rows, c2 + 40), device="cuda", dtype=dtype)
    w1[:, 16:16 + c1] = h1
    w2[:, 8:8 + c2] = h2
    y2 = ops.groupnorm(w1[:, 16:16 + c1], samples, rows, gamma, beta, 1e-5, True, x2=w2[:, 8:8 + c2])
    _check_gn(y2, xc, samples, rows, 32, gamma, beta, 1e-5, True, "two-pass concat")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c,groups,rows", [(320, 32, 128), (320, 32, 128 * 64), (64, 4, 1024), (256, 4, 128 * 3)])
def test_groupnorm_column_statistics(dtype, c, groups, rows):
    """gn_finalize_kernel: tps * cpg = 10 (< 32 threads), 640 (> 256 threads, each thread walking several pairs), and
    4 groups (16 / 64 channels per group) against float64."""
    from animate_anything_b200 import ops
    samples = 3
    tps, cpg = rows // 128, c // groups
    assert (tps * cpg < 32) or (tps * cpg > 256) or groups != 32
    gamma, beta = _affine(c, 5)
    h = _producer(samples * rows, c, dtype, c + rows, shift=0.4)
    y = ops.groupnorm(h, samples, rows, gamma, beta, 1e-6, True, groups)
    _check_gn(y, h, samples, rows, groups, gamma, beta, 1e-6, True, (c, groups, rows))
    assert torch.equal(y, ops.groupnorm(h, samples, rows, gamma, beta, 1e-6, True, groups))


@pytest.mark.parametrize("dtype", DTYPES)
def test_groupnorm_strided_input(dtype):
    """A column slice of a wider tensor (offset 8 elements, row stride C + 24), both with and without SiLU."""
    from animate_anything_b200 import ops
    samples, rows, c = 2, 300, 320
    wide = _randn((samples * rows, c + 24), dtype, 7, 1.5, 0.3)
    x = wide[:, 8:8 + c]
    gamma, beta = _affine(c, 8)
    for silu in (True, False):
        y = ops.groupnorm(x, samples, rows, gamma, beta, 1e-5, silu)
        _check_gn(y, x, samples, rows, 32, gamma, beta, 1e-5, silu, silu)


@pytest.mark.parametrize("dtype", DTYPES)
def test_groupnorm_workspace_sample_counts(dtype):
    """Calls with different sample counts (up to the 4096 the ticket header holds) alternate through the one shared
    workspace; each repeated call gives the same bits, and 4097 samples are rejected."""
    from animate_anything_b200 import _lib, ops
    gamma, beta = _affine(320, 9)
    seq = [(3, 100, 320), (4096, 16, 320), (1, 1000, 320), (4096, 8, 64), (7, 64, 320), (2, 4096, 320)]
    for i, (samples, rows, c) in enumerate(seq):
        x = _randn((samples * rows, c), dtype, 30 + i, 1.5, 0.3)
        y = ops.groupnorm(x, samples, rows, gamma[:c], beta[:c], 1e-5, True)
        assert torch.equal(y, ops.groupnorm(x, samples, rows, gamma[:c], beta[:c], 1e-5, True)), (samples, rows, c)
        _check_gn(y, x, samples, rows, 32, gamma[:c], beta[:c], 1e-5, True, (samples, rows, c))
    x = _randn((4097 * 8, 64), dtype, 40)
    with pytest.raises(_lib.AabError):
        ops.groupnorm(x, 4097, 8, gamma[:64], beta[:64], 1e-5, True)


@pytest.mark.parametrize("dtype", DTYPES)
def test_groupnorm_large_mean(dtype):
    """mean / std = 10, 50, 200 (and the ratios between) through both paths: the same GEMM output, with and without its
    column statistics.  Both stay inside the bound of `_gn_bound`, whose cancellation term grows as r^2 * 2^-18 * |z|.
    The output shows, per path, the largest error in units of one output rounding, over all outputs and over those with
    |z| >= 1.  Near zero the output ulp is far below the fp32 error of the apply pass itself (~2^-24 (r + 1)), so the
    ratio at which the statistics leave the one-ulp bound is read from the |z| >= 1 column."""
    from animate_anything_b200 import ops
    samples, rows, c = 2, 4096, 320
    gamma = torch.ones(c, device="cuda")
    beta = torch.zeros(c, device="cuda")
    worst = {}
    for ratio in (1, 2, 5, 10, 20, 50, 100, 200):
        h = _producer(samples * rows, c, dtype, 50 + ratio, shift=ratio)
        ref, z, r = _gn_ref(h, samples, rows, 32, gamma, beta, 1e-5, False)
        ulp = _ulp(ref, dtype)
        tol = _gn_bound(ref, z, r, gamma, beta, False, dtype)
        for path, y in (("colstats", ops.groupnorm(h, samples, rows, gamma, beta, 1e-5, False)),
                        ("two-pass", ops.groupnorm(h.clone(), samples, rows, gamma, beta, 1e-5, False))):
            err = (y.double() - ref).abs()
            assert bool((err <= tol).all()), (path, ratio, float((err / tol).max()))
            worst[(path, ratio)] = (float((err / ulp).max()), float((err / ulp)[z.abs() >= 1].max()))
    for path in ("two-pass", "colstats"):
        row = "  ".join(f"r={k[1]}: {v[0]:.2f} / {v[1]:.2f}" for k, v in worst.items() if k[0] == path)
        first = next((k[1] for k, v in worst.items() if k[0] == path and v[1] > 1.0), None)
        print(f"groupnorm {dtype} {path}: max error / output ulp (all / |z| >= 1)  {row}  -> |z| >= 1 leaves one ulp at "
              f"r = {first}")
    # the column statistics must not be clearly worse than the two-pass statistics at a ratio the models can reach
    assert worst[("colstats", 50)][0] <= 2 * worst[("two-pass", 50)][0] + 1.0, worst


# ---------------------------------------------------------------------------------------------- LayerNorm
# one C per dispatch instance <OPL, LPR> of aab_layernorm, including both sides of every boundary:
# 8, 64 -> <1,8>; 72, 128 -> <2,8>; 192 <3,8>; 256 <4,8>; 320 <5,8>; 512 <4,16>; 640 <5,16>; 1024 <4,32>; 1280 <5,32>;
# 2048 <8,32>
LN_C = [8, 64, 72, 128, 192, 256, 320, 512, 640, 1024, 1280, 2048]


def _ln_rows_per_warp(c):
    v = c // 8
    lpr = 8 if v <= 40 else (16 if v <= 80 else 32)
    return 32 // lpr


def _ln_check(y, x, gamma, beta, eps, what):
    """fp32 LayerNorm: the mean is a sum of C values in per-lane chains of <= 64 terms plus a shuffle tree (relative error
    < 2^-18 of sum |x|), the variance is an exact two-pass sum of squared deviations, rsqrtf is within 2 ulp: the normalised
    value z carries an error below 2^-17 * (|z| + mean|x| / std), then (v - mean) * rstd * gamma + beta adds a few fp32
    roundings of |gamma * z| and |beta|."""
    c = x.shape[1]
    xd = x.double()
    ref = F.layer_norm(xd, (c,), gamma.double(), beta.double(), eps)
    std = torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + eps)
    z = (xd - xd.mean(-1, keepdim=True)) / std
    rr = xd.abs().mean(-1, keepdim=True) / std
    g = gamma.double().abs()
    tol = _ulp(ref, y.dtype) + 2.0 ** -17 * (g * (z.abs() + rr + 1) + beta.double().abs())
    err = (y.double() - ref).abs()
    assert bool((err <= tol).all()), (what, float((err / tol).max()))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", LN_C)
def test_layernorm_instances(dtype, c):
    """Rows 1, 3, a count that leaves the last warp's row group partly filled, and one row past what the persistent grid
    covers in one sweep (6 CTAs x 8 warps per SM, each warp 32 / LPR rows)."""
    from animate_anything_b200 import _lib, ops
    rpw = _ln_rows_per_warp(c)
    sweep = 6 * _lib.load().aab_num_sms() * 8 * rpw
    gamma, beta = _affine(c, c)
    for rows in (1, 3, 4 * 77 + 1 if rpw > 1 else 1001, sweep + 1):
        assert rows % rpw or rpw == 1 or rows == 1
        x = _randn((rows, c), dtype, rows + c, 2.0, 0.5)
        y = ops.layernorm(x, gamma, beta, 1e-5)
        _ln_check(y, x, gamma, beta, 1e-5, (c, rows))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", LN_C)
def test_layernorm_constant_row_gives_beta(dtype, c):
    """A row of identical values (zero, powers of two, 3 and -1.25: C * v * fp32(1/C) == v, so the fp32 mean is exact)
    has zero deviation: the output is exactly beta rounded to the output type."""
    from animate_anything_b200 import ops
    gamma, beta = _affine(c, c + 1)
    vals = torch.tensor([0.0, 1.0, -2.0, 3.0, -1.25], device="cuda")
    x = vals[:, None].expand(5, c).to(dtype).contiguous()
    y = ops.layernorm(x, gamma, beta, 1e-5)
    assert torch.equal(y, beta.to(dtype).expand(5, c))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c,l", [(1280, 257), (1024, 77), (64, 5)])
def test_layernorm_token0_rows(dtype, c, l):
    """The pooled LayerNorm of the CLIP vision tower: token 0 of every sequence, rows `l * c` apart."""
    from animate_anything_b200 import ops
    b = 3
    last = _randn((b, l, c), dtype, c + l, 2.0, 0.5)
    gamma, beta = _affine(c, 11)
    x = last[:, 0]
    assert x.stride(0) == l * c
    y = ops.layernorm(x, gamma, beta, 1e-5)
    _ln_check(y, x, gamma, beta, 1e-5, (c, l))


# ---------------------------------------------------------------------------------------------- row softmax
def _softmax_rows(s, dtype, pad, prefill=math.nan):
    """aab_softmax_rows into a buffer pre-filled with `prefill`, probability rows `pad` wide."""
    from animate_anything_b200 import _lib
    p = torch.full((s.shape[0], pad), prefill, device="cuda", dtype=dtype)
    _lib.call("aab_softmax_rows", C.c_void_p(s.data_ptr()), s.stride(0), C.c_void_p(p.data_ptr()), p.stride(0), s.shape[0],
              s.shape[1], int(dtype == torch.bfloat16), _stream())
    return p


def _logit_patterns(l, seed):
    g = _gen(seed)
    base = torch.randn((8, l), device="cuda", generator=g) * 3
    base[0, 0] = base[0].max() + 5                   # row maximum first
    base[1, -1] = base[1].max() + 5                  # last
    base[2, l // 2] = base[2].max() + 5              # middle
    base[3] = 0.0
    base[3, (7 * l) // 11] = 40.0                    # one dominant logit
    base[4] = 1.7                                    # all equal
    base[5] = torch.rand(l, device="cuda", generator=g) * 100 - 50   # spread 100: most terms underflow
    if l > 1:
        base[6, 1::3] = -math.inf                    # -inf entries -> exactly 0
        base[7, :-1] = -math.inf
    return base


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("l", [1, 7, 9, 255, 256, 257, 1000, 4096])
def test_softmax_rows_padding_and_patterns(dtype, l):
    """float64 softmax of the fp32 scores (strided: lds = L + 13); the pad columns L..ceil8(L)-1 are exactly +0 although the
    buffer held NaN; -inf logits give exactly 0.
    Slack: exp is __expf (ex2.approx of s * log2 e: a relative error of about 2^-22 * (2 + |s - max|)), the sum adds L such
    terms in per-thread chains of L / 256 plus a 256-way tree (relative error < 2^-18), 1 / sum is correctly rounded; and
    __expf flushes results below 2^-126 to zero, an absolute error of at most the smallest normal fp32 value."""
    from animate_anything_b200 import ops
    pad = (l + 7) // 8 * 8
    wide = torch.full((8, l + 13), 7.0, device="cuda")
    wide[:, :l] = _logit_patterns(l, l)
    s = wide[:, :l]
    for what, p in (("nan-filled", _softmax_rows(s, dtype, pad)), ("ops.softmax_rows", ops.softmax_rows(s, dtype, pad_to=pad))):
        assert p.shape == (8, pad)
        assert torch.equal(p[:, l:].view(torch.int16), torch.zeros((8, pad - l), device="cuda", dtype=torch.int16)), what
        sd = s.double()
        ref = torch.softmax(sd, -1)
        err = (p[:, :l].double() - ref).abs()
        gap = (sd.max(-1, keepdim=True).values - sd).nan_to_num(posinf=0.0)
        tol = _ulp(ref, dtype) + ref * 2.0 ** -22 * (16 + gap) + torch.finfo(torch.float32).tiny
        assert bool((err <= tol).all()), (what, float((err / tol).max()))
        assert bool((p[:, :l][torch.isinf(s)] == 0).all())
    if l > 1:
        assert float(p[7, l - 1]) == 1.0


# ---------------------------------------------------------------------------------------------- VAE mid-block attention
def _attn_ref(qkv, n, l, c):
    """float64 softmax(Q K^T / sqrt(c)) V per frame, the float64 probabilities, |Q| |K|^T / sqrt(c) and V."""
    t = qkv.double().reshape(n, l, 3 * c)
    q, k, v = t[..., :c], t[..., c:2 * c], t[..., 2 * c:]
    p = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(c), -1)
    return (p @ v).reshape(n * l, c), p, (q.abs() @ k.abs().transpose(1, 2)) / math.sqrt(c), v


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", [128, 512])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("l", [64, 100, 130, 1024])
def test_vae_mid_attention_chain(dtype, c, n, l):
    """ops.single_head_attention (Q.K^T batched GEMM, padded row softmax, transpose, P.V batched GEMM) against float64.
    Bound: one rounding of the output, plus the 16-bit rounding of each probability (half an ulp of P_j, times |v_j|),
    plus the fp32 error of the scores (2^-18 of sum |q||k| / sqrt(c), moving P_j by that much relative) and of the P.V
    accumulation (2^-18 of sum P_j |v_j|).  With n = 3: changing frame 1's K and V leaves frame 0 unchanged bit for bit."""
    from animate_anything_b200 import ops
    qkv = _randn((n * l, 3 * c), dtype, c + l + n)
    o = ops.single_head_attention(qkv, n, l, c)
    assert o.shape == (n * l, c)
    ref, p, qk, v = _attn_ref(qkv, n, l, c)
    a = _ulp(p, dtype) / 2 + p * 2.0 ** -18 * (1 + qk)
    tol = _ulp(ref, dtype) + (a @ v.abs()).reshape(n * l, c) + 2.0 ** -18 * (p @ v.abs()).reshape(n * l, c)
    err = (o.double() - ref).abs()
    assert bool((err <= tol).all()), float((err / tol).max())
    if n > 1:
        qkv2 = qkv.clone()
        qkv2[l:2 * l, c:] = _randn((l, 2 * c), dtype, 99)
        o2 = ops.single_head_attention(qkv2, n, l, c)
        assert torch.equal(o2[:l], o[:l]) and torch.equal(o2[2 * l:], o[2 * l:])
        assert not torch.equal(o2[l:2 * l], o[l:2 * l])
