"""GPU: the attention kernels at the lengths, score patterns and arguments where flash attention goes wrong, against float64
softmax attention on the same 16-bit inputs."""
import ctypes as C
import math

import pytest
import torch

from util import check

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
TOL = {torch.float16: (2e-3, 2e-3), torch.bfloat16: (1.6e-2, 1.6e-2)}
LOG2E = 1.4426950408889634


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def _ref(q, k, v, scale, causal=False):
    """float64 softmax attention; q [B, H, Lq, D], k / v [B, H, Lk, D]."""
    s = torch.einsum("bhqd,bhkd->bhqk", q.double(), k.double()) * scale
    if causal:
        lq, lk = s.shape[-2:]
        s = s.masked_fill(torch.ones(lq, lk, dtype=torch.bool, device=s.device).triu(1), -math.inf)
    return torch.einsum("bhqk,bhkd->bhqd", torch.softmax(s, dim=-1), v.double())


def _heads(x, nb, l, heads, d):
    return x.reshape(nb, l, heads, d).permute(0, 2, 1, 3)


def _unheads(x):
    nb, heads, l, d = x.shape
    return x.permute(0, 2, 1, 3).reshape(nb * l, heads * d)


def _d64(q, kv, nb, lq, lk, heads, div=1, scale=0.125, causal=False, d=64):
    """Run the kernel (head dim 64 or 80) on q [nb*lq, H*d], kv [nb_kv*lk, 2*H*d] (K then V) and build the reference."""
    from animate_anything_b200 import ops
    c = heads * d
    if d == 64:
        out = ops.flash_attn_d64(q, 0, kv, 0, c, nb, lq, lk, heads, kv_batch_div=div, causal=causal, scale=scale)
    else:
        out = ops.flash_attn_d80(q, 0, kv, 0, c, nb, lq, lk, heads, kv_batch_div=div, scale=scale)
    torch.cuda.synchronize()
    nb_kv = kv.shape[0] // lk
    kb = torch.arange(nb, device="cuda") // div
    k = _heads(kv[:, :c], nb_kv, lk, heads, d)[kb]
    v = _heads(kv[:, c:], nb_kv, lk, heads, d)[kb]
    return out, _unheads(_ref(_heads(q, nb, lq, heads, d), k, v, scale, causal))


# ---------------------------------------------------------------------------------------------- flash d64: lengths
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lq", [1, 77, 127, 128, 129])
@pytest.mark.parametrize("lk", [1, 8, 63, 64, 65, 127, 128, 129, 192, 193])
def test_flash_d64_tail_lengths(dtype, lq, lk):
    nb, heads = 2, 2
    q = _rand((nb * lq, heads * 64), dtype, lq, 1.5)
    kv = _rand((nb * lk, 2 * heads * 64), dtype, 1000 + lk, 1.5)
    out, ref = _d64(q, kv, nb, lq, lk, heads)
    check(f"flash d64 lq{lq} lk{lk} {dtype}", out, ref, *TOL[dtype])


# ---------------------------------------------------------------------------------------------- flash d64: score patterns
def _biased(nb, lq, lk, heads, dtype, bias, seed, d=64):
    """q / kv whose scores are score_ij = (4 * bias_j + noise_ij) * scale: dimension 0 of every query is 4 and dimension 0
    of key j is bias_j (16-bit), the other dimensions are random."""
    c = heads * d
    q = _rand((nb * lq, c), dtype, seed)
    kv = _rand((nb * lk, 2 * c), dtype, seed + 1)
    q.view(nb * lq, heads, d)[:, :, 0] = 4.0
    kv.view(nb, lk, 2, heads, d)[:, :, 0, :, 0] = bias.to(dtype).view(1, lk, 1)
    return q, kv


def _pattern(name, lk, seed):
    """Per-key bias; 4 * bias * (1/8) * log2(e) spans about 45 in log2 units (x 1.4 for the staircase)."""
    j = torch.arange(lk, device="cuda", dtype=torch.float64)
    span = 62.0
    if name == "max_first":                  # row maximum in block 0, then ever smaller
        return -span * j / max(lk - 1, 1)
    if name == "max_last":                   # maximum in the last (partially masked) block: the running max jumps late
        return span * j / max(lk - 1, 1)
    if name == "staircase":                  # every 64-key block raises the running max by ~14 in log2: a rescale per block
        g = torch.Generator(device="cuda").manual_seed(seed)
        return 20.0 * torch.div(j, 64, rounding_mode="floor") + torch.rand(lk, device="cuda", generator=g, dtype=torch.float64)
    if name in ("onehot_first", "onehot_last"):
        b = torch.full((lk,), -span / 2, device="cuda", dtype=torch.float64)
        b[0 if name == "onehot_first" else lk - 1] = span / 2
        return b
    raise ValueError(name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pattern", ["max_first", "max_last", "staircase", "onehot_first", "onehot_last"])
@pytest.mark.parametrize("lk", [65, 129, 193, 200])
def test_flash_d64_large_logit_patterns(dtype, pattern, lk):
    nb, heads, lq = 2, 2, 129
    q, kv = _biased(nb, lq, lk, heads, dtype, _pattern(pattern, lk, lk), lk)
    out, ref = _d64(q, kv, nb, lq, lk, heads)
    check(f"flash d64 {pattern} lk{lk} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lk", [1, 63, 65, 193])
def test_flash_d64_all_keys_equal(dtype, lk):
    """Identical keys: the softmax is uniform over exactly lk keys, the output is the mean of V (masked keys excluded)."""
    nb, heads, lq = 2, 2, 77
    c = heads * 64
    q = _rand((nb * lq, c), dtype, 1, 3.0)
    kv = _rand((nb * lk, 2 * c), dtype, 2)
    kv[:, :c] = _rand((1, c), dtype, 3, 3.0)
    out, ref = _d64(q, kv, nb, lq, lk, heads)
    mean = _unheads(_heads(kv[:, c:], nb, lk, heads, 64).double().mean(dim=2, keepdim=True).expand(nb, heads, lq, 64))
    check(f"flash d64 equal keys lk{lk} {dtype}", out, ref, *TOL[dtype])
    check(f"flash d64 equal keys = mean(V) lk{lk} {dtype}", out, mean, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lk", [1, 63, 65, 127, 129])
def test_flash_d64_no_leakage_past_lk(dtype, lk):
    """K/V rows just past Lk belong to the next batch (or are TMA zero fill after the last one).  Filling the next batches
    with keys that would win every softmax and huge values changes nothing in batch 0, bit for bit."""
    nb, heads, lq = 3, 2, 77
    c = heads * 64
    q = _rand((nb * lq, c), dtype, 1)
    q.view(nb * lq, heads, 64)[:, :, 0] = 4.0
    kv = _rand((nb * lk, 2 * c), dtype, 2)
    out, ref = _d64(q, kv, nb, lq, lk, heads)
    loud = kv.clone()
    loud[lk:, :c] = 0.5
    loud.view(nb * lk, 2, heads, 64)[lk:, 0, :, 0] = 1000.0
    loud[lk:, c:] = 30000.0
    out_loud, _ = _d64(q, loud, nb, lq, lk, heads)
    alone, _ = _d64(q[:lq].contiguous(), kv[:lk].contiguous(), 1, lq, lk, heads)
    check(f"flash d64 leakage lk{lk} {dtype}", out, ref, *TOL[dtype])
    assert torch.equal(out_loud[:lq], out[:lq]) and torch.equal(alone, out[:lq])


# ---------------------------------------------------------------------------------------------- flash d64: other arguments
@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_d64_scale_and_kv_batch_div(dtype):
    nb, heads, lq, lk = 6, 3, 77, 129
    q = _rand((nb * lq, heads * 64), dtype, 1)
    kv = _rand((2 * lk, 2 * heads * 64), dtype, 2)
    out, ref = _d64(q, kv, nb, lq, lk, heads, div=3, scale=0.3)
    check(f"flash d64 scale 0.3 div 3 {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_d64_strided_output(dtype):
    """`out` with a row stride wider than the heads, a nonzero out_col0 and a batch stride larger than lq rows: the heads land
    in their columns and nothing else in the buffer is written."""
    from animate_anything_b200 import _lib
    nb, heads, lq, lk, col0 = 2, 2, 77, 129, 40
    c = heads * 64
    q = _rand((nb * lq, c), dtype, 1)
    kv = _rand((nb * lk, 2 * c), dtype, 2)
    ld_out, rows_per_batch = c + 72, lq + 3
    buf = torch.full((nb * rows_per_batch, ld_out), -5.0, device="cuda", dtype=dtype)
    want = buf.clone()
    _, ref = _d64(q, kv, nb, lq, lk, heads)
    _lib.call("aab_flash_attn_d64", C.c_void_p(q.data_ptr()), c, lq * c, c, 0, C.c_void_p(kv.data_ptr()), 2 * c, lk * 2 * c, 2 * c,
              0, c, C.c_void_p(buf.data_ptr()), ld_out, rows_per_batch * ld_out, col0, nb, nb, 1, heads, lq, lk, 0.125,
              int(dtype == torch.bfloat16), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    got = buf.view(nb, rows_per_batch, ld_out)[:, :lq, col0:col0 + c].reshape(nb * lq, c)
    check(f"flash d64 strided out {dtype}", got, ref, *TOL[dtype])
    want.view(nb, rows_per_batch, ld_out)[:, :lq, col0:col0 + c] = got.view(nb, lq, c)
    assert torch.equal(buf, want)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("l", [1, 2, 63, 64, 65, 77, 128])
def test_flash_d64_causal(dtype, l):
    from animate_anything_b200 import ops
    nb, heads = 2, 3
    c = heads * 64
    qkv = _rand((nb * l, 3 * c), dtype, l, 1.5)
    out = ops.flash_attn_d64(qkv, 0, qkv, c, 2 * c, nb, l, l, heads, causal=True)
    torch.cuda.synchronize()
    t = qkv.reshape(nb, l, 3, heads, 64).permute(2, 0, 3, 1, 4)
    check(f"flash d64 causal l{l} {dtype}", out, _unheads(_ref(t[0], t[1], t[2], 0.125, causal=True)), *TOL[dtype])


# ---------------------------------------------------------------------------------------------- flash d80
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lq", [1, 77, 257])
@pytest.mark.parametrize("lk", [1, 31, 32, 33, 63, 64, 65, 129, 257])
def test_flash_d80_tail_lengths(dtype, lq, lk):
    nb, heads = 2, 2
    q = _rand((nb * lq, heads * 80), dtype, lq)
    kv = _rand((nb * lk, 2 * heads * 80), dtype, 1000 + lk)
    out, ref = _d64(q, kv, nb, lq, lk, heads, scale=80 ** -0.5, d=80)
    check(f"flash d80 lq{lq} lk{lk} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pattern", ["max_last", "staircase"])
@pytest.mark.parametrize("lk", [33, 65, 257])
def test_flash_d80_large_logit_patterns(dtype, pattern, lk):
    nb, heads, lq = 2, 2, 129
    q, kv = _biased(nb, lq, lk, heads, dtype, _pattern(pattern, lk, lk) * (80 ** 0.5 / 8), lk, d=80)
    out, ref = _d64(q, kv, nb, lq, lk, heads, scale=80 ** -0.5, d=80)
    check(f"flash d80 {pattern} lk{lk} {dtype}", out, ref, *TOL[dtype])


# ---------------------------------------------------------------------------------------------- temporal attention
def _temporal(qkv, b, t, hw, heads):
    from animate_anything_b200 import ops
    c = heads * 64
    out = ops.temporal_attn_d64(qkv, b, t, hw, heads, 0, c, 2 * c)
    torch.cuda.synchronize()
    x = qkv.reshape(b, t, hw, 3, heads, 64).permute(3, 0, 2, 4, 1, 5).reshape(3, b * hw, heads, t, 64)
    ref = _ref(x[0], x[1], x[2], 0.125).reshape(b, hw, heads, t, 64).permute(0, 3, 1, 2, 4).reshape(b * t * hw, c)
    return out, ref


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("t", [1, 2, 15, 16, 17, 31, 32])
def test_temporal_frame_counts(dtype, t):
    b, hw, heads = 2, 24, 2
    qkv = _rand((b * t * hw, 3 * heads * 64), dtype, t, 1.5)
    out, ref = _temporal(qkv, b, t, hw, heads)
    check(f"temporal t{t} {dtype}", out, ref, *TOL[dtype])


def test_temporal_rejects_33_frames():
    from animate_anything_b200 import _lib, ops
    qkv = torch.zeros((33 * 4, 3 * 64), device="cuda", dtype=torch.float16)
    with pytest.raises(_lib.AabError, match="status 1"):
        ops.temporal_attn_d64(qkv, 1, 33, 4, 1, 0, 64, 128)


def _persistent_shape():
    """(b, t, hw, heads) with at least four (b, pixel, head) items per warp of the persistent grid (two 4-warp CTAs per SM)
    and a total that is not a multiple of the grid stride, so that every warp reuses its first buffer and the last round
    is ragged."""
    from animate_anything_b200 import _lib
    b, t, hw, heads = 2, 14, 1100, 2
    total = b * hw * heads
    stride = min((total + 3) // 4, 2 * _lib.load().aab_num_sms()) * 4
    assert total >= 4 * stride and total % stride != 0, (total, stride)
    return b, t, hw, heads


@pytest.mark.parametrize("dtype", DTYPES)
def test_temporal_persistent_loop(dtype):
    b, t, hw, heads = _persistent_shape()
    qkv = _rand((b * t * hw, 3 * heads * 64), dtype, 5)
    out, ref = _temporal(qkv, b, t, hw, heads)
    check(f"temporal persistent b{b} t{t} hw{hw} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("t", [17, 32])
@pytest.mark.parametrize("pattern", ["max_last", "onehot_last", "max_first"])
def test_temporal_large_logits(dtype, t, pattern):
    b, hw, heads = 2, 40, 2
    c = heads * 64
    qkv = _rand((b * t * hw, 3 * c), dtype, t)
    v = qkv.view(b, t, hw, 3, heads, 64)
    v[:, :, :, 0, :, 0] = 4.0
    v[:, :, :, 1, :, 0] = _pattern(pattern, t, t).to(dtype).view(1, t, 1, 1)
    out, ref = _temporal(qkv, b, t, hw, heads)
    check(f"temporal {pattern} t{t} {dtype}", out, ref, *TOL[dtype])

