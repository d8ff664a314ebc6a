"""The staged epilogue of the implicit GEMM (output tile staged in shared memory and stored by TMA, residual loaded by TMA,
column statistics taken by the producer warpgroup's spare warps): every width with a ragged last n-tile, a partial last
m-tile, column slices of the output and the residual, the two-source concat, per-sample bias, GEGLU, two CTAs per SM, and
the layouts the host routes to the per-element epilogue.  Results against torch; column statistics against float64 sums
of the kernel's own output; without an activation the staged result is bit-identical to the per-element epilogue."""
import pytest
import torch
import torch.nn.functional as F

from util import check

pytestmark = pytest.mark.gpu

TOL = {torch.float16: (1e-3, 1e-4), torch.bfloat16: (8e-3, 8e-4)}
DTYPES = [torch.float16, torch.bfloat16]


def _ops():
    from animate_anything_b200 import ops
    return ops


def _rand(shape, dtype, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def _check_stats(name, out, rows_per_tile=128):
    st = getattr(out, "_aab_stats", None)
    assert st is not None, f"{name}: no column statistics"
    m, n = out.shape
    o = torch.zeros((st.shape[0] * rows_per_tile, n), dtype=torch.float64, device=out.device)
    o[:m] = out.double()
    o = o.reshape(st.shape[0], rows_per_tile, n)
    check(f"{name} colstats sum", st[..., 0], o.sum(1).float(), 1e-5, 1e-3)
    check(f"{name} colstats sumsq", st[..., 1], (o * o).sum(1).float(), 1e-5, 1e-3)


# N = 288 leaves a ragged last n-tile at every width; 3400 rows = 26 full m-tiles + 72 rows (column statistics are only
# requested where every m-tile is whole)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bn", [64, 128, 160, 192, 256])
@pytest.mark.parametrize("m", [3456, 3400])
def test_widths_ragged(dtype, bn, m):
    ops = _ops()
    k, n = 320, 288
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    res = _rand((m, n), dtype, 1.0, 4)
    b2 = _rand((-(-m // 500), n), torch.float32, 1.0, 5)
    ref = x.float() @ w.float().t() + b
    cases = {"plain": ({}, ref), "residual": ({"residual": res}, ref + res.float()),
             "bias2": ({"bias2": b2, "rows_per_bias2": 500}, ref + b2.repeat_interleave(500, dim=0)[:m]),
             "silu": ({"act": ops.ACT_SILU}, F.silu(ref))}
    for name, (kw, r) in cases.items():
        out = ops.linear(x, w, b, block_n=bn, ctas_per_sm=1, stats=True, **kw)
        check(f"bn {bn} {name} {dtype}", out, r, *TOL[dtype])
        if m % 128 == 0:
            _check_stats(f"bn {bn} {name}", out)
        if name != "silu":
            assert torch.equal(out, ops.linear(x, w, b, block_n=bn, ctas_per_sm=1, direct=True, **kw)), name


@pytest.mark.parametrize("dtype", DTYPES)
def test_column_slices(dtype):
    """Output and residual are column slices of wider tensors, with ld_out != ld_res != n_out."""
    ops = _ops()
    m, k, n = 2176, 256, 320
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    res_big = _rand((m, 2 * n + 64), dtype, 1.0, 4)
    res = res_big[:, 64:64 + n]
    out_big = torch.full((m, n + 96), 7.0, device="cuda", dtype=dtype)
    out = out_big[:, 32:32 + n]
    got = ops.linear(x, w, b, out=out, residual=res, stats=True)
    assert got.data_ptr() == out.data_ptr()
    check(f"slices {dtype}", out, x.float() @ w.float().t() + b + res.float(), *TOL[dtype])
    assert bool((out_big[:, :32] == 7).all()) and bool((out_big[:, 32 + n:] == 7).all()), "wrote outside the slice"
    _check_stats("slices", got)
    ref_direct = torch.empty_like(out_big)
    ops.linear(x, w, b, out=ref_direct[:, 32:32 + n], residual=res, direct=True)
    assert torch.equal(out, ref_direct[:, 32:32 + n])


@pytest.mark.parametrize("dtype", DTYPES)
def test_two_source_concat_and_conv(dtype):
    ops = _ops()
    m, c1, c2, n = 4096, 192, 128, 320
    x = _rand((m, c1), dtype, 1.0, 1)
    x2 = _rand((m, c2), dtype, 1.0, 2)
    w = _rand((n, c1 + c2), dtype, (c1 + c2) ** -0.5, 3)
    b = _rand((n,), torch.float32, 1.0, 4)
    res = _rand((m, n), dtype, 1.0, 5)
    out = ops.conv1x1_cat(x, x2, w, b, residual=res, stats=True)
    check(f"concat {dtype}", out, torch.cat([x, x2], 1).float() @ w.float().t() + b + res.float(), *TOL[dtype])
    _check_stats("concat", out)
    # conv3x3 at a width the box does not divide (partial rows inside every tile) with a per-frame bias
    nb, h, wd, c = 4, 24, 40, 64
    xi = _rand((nb, h, wd, c), dtype, 1.0, 6)
    wc = _rand((n, 9 * c), dtype, (9 * c) ** -0.5, 7)
    b2 = _rand((nb, n), torch.float32, 1.0, 8)
    got = ops.conv3x3(xi, wc, b, bias2=b2, rows_per_bias2=h * wd)
    ref = F.conv2d(xi.permute(0, 3, 1, 2).float(), wc.float().view(n, 3, 3, c).permute(0, 3, 1, 2), b, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, n) + b2.repeat_interleave(h * wd, dim=0)
    check(f"conv3x3 bias2 {dtype}", got, ref, *TOL[dtype])
    assert torch.equal(got, ops.conv3x3(xi, wc, b, bias2=b2, rows_per_bias2=h * wd, direct=True))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n_out", [64, 320])
def test_geglu(dtype, n_out):
    ops = _ops()
    m, k = 3400, 320
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((2 * n_out, k), dtype, k ** -0.5, 2)
    b = _rand((2 * n_out,), torch.float32, 1.0, 3)
    out = ops.linear(x, w, b, geglu=True)
    hv = x.float() @ w.float().t() + b
    ref = hv[:, :n_out] * F.gelu(hv[:, n_out:])
    check(f"geglu {n_out} {dtype}", out, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
def test_two_cta(dtype):
    ops = _ops()
    m, k, n = 139264, 320, 320                   # more m-tiles than two per SM
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    res = _rand((m, n), dtype, 1.0, 4)
    two = ops.linear(x, w, b, residual=res, block_n=64, ctas_per_sm=2, stats=True)
    check(f"two-cta {dtype}", two, x.float() @ w.float().t() + b + res.float(), *TOL[dtype])
    _check_stats("two-cta", two)
    one = ops.linear(x, w, b, residual=res, block_n=64, ctas_per_sm=1, stats=True)
    assert torch.equal(two, one) and torch.equal(two._aab_stats, one._aab_stats)


@pytest.mark.parametrize("dtype", DTYPES)
def test_layouts_routed_to_direct(dtype):
    """Layouts a TMA box cannot address take the per-element epilogue: still right, and no column statistics."""
    ops = _ops()
    m, k, n = 1000, 128, 256
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    res_big = _rand((m, n + 4), dtype, 1.0, 4)
    ref = x.float() @ w.float().t() + b
    # output rows 2 * (n + 4) bytes apart: not a multiple of 16
    big = torch.empty((m, n + 4), device="cuda", dtype=dtype)
    out = ops.linear(x, w, b, out=big[:, :n], stats=True)
    check(f"ld_out {dtype}", big[:, :n], ref, *TOL[dtype])
    assert getattr(out, "_aab_stats", None) is None
    # output base 8 bytes past a 16-byte boundary
    big = torch.empty((m, n + 8), device="cuda", dtype=dtype)
    out = ops.linear(x, w, b, out=big[:, 4:4 + n], stats=True)
    check(f"misaligned out {dtype}", big[:, 4:4 + n], ref, *TOL[dtype])
    assert getattr(out, "_aab_stats", None) is None
    # residual rows not a multiple of 16 bytes apart
    out = ops.linear(x, w, b, residual=res_big[:, :n], stats=True)
    check(f"ld_res {dtype}", out, ref + res_big[:, :n].float(), *TOL[dtype])
    assert getattr(out, "_aab_stats", None) is None
    # a per-sample bias whose samples are shorter than a tile (more than two samples per tile)
    b2 = _rand((-(-m // 100), n), torch.float32, 1.0, 5)
    out = ops.linear(x, w, b, bias2=b2, rows_per_bias2=100, stats=True)
    check(f"short samples {dtype}", out, ref + b2.repeat_interleave(100, dim=0)[:m], *TOL[dtype])
    assert getattr(out, "_aab_stats", None) is None
