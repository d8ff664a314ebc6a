"""Fitted tile widths (160 / 192 columns) and the slab epilogue of the implicit GEMM: every output and column-statistics
table is bit-identical to the same launch forced to 64-column tiles (the K order of an element does not depend on the
width), and within the 16-bit rounding of the fp32 torch reference."""
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


def _launched_widths(ops, fn):
    """Run fn() and return (result, tile widths of the implicit-GEMM launches it made)."""
    ops.IGEMM_PROFILE = []
    try:
        out = fn()
        widths = [p["block_n"] for p in ops.IGEMM_PROFILE]
    finally:
        ops.IGEMM_PROFILE = None
    return out, widths


def _same(name, fitted, narrow):
    assert torch.equal(fitted, narrow), f"{name}: fitted width differs from 64-column tiles"
    sf, sn = getattr(fitted, "_aab_stats", None), getattr(narrow, "_aab_stats", None)
    assert (sf is None) == (sn is None), name
    if sf is not None:
        assert torch.equal(sf, sn), f"{name}: column statistics differ"


def test_fit_rule_on_132_sms():
    ops = _ops()
    fit = lambda n, m: ops.fit_block_n(n, m, 132)
    assert fit(320, 1088) == 160 and fit(640, 272) == 160
    assert fit(960, 1088) == 192 and fit(1920, 272) == 192
    assert fit(1280, 68) == 256 and fit(1280, 17) == 192
    assert fit(128, 8192) == 256 and fit(256, 4096) == 256


def _fitted(ops, n, m_tiles):
    return ops.fit_block_n(n, m_tiles, ops._lib.load().aab_num_sms())


# On 132 SMs these take 160, 160, 192, 192 and 192 columns (2176 rows = 17 m-tiles); 34788, 3400 and 17400 rows end in a
# partial m-tile.  N = 328 is a width no tile divides and n % 32 != 0: per-element stores.
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m,k,n", [(34788, 320, 320), (3400, 640, 640), (17400, 320, 960), (34816, 320, 1920),
                                   (2176, 1280, 1280), (139, 512, 328)])
def test_linear_widths(dtype, m, k, n):
    ops = _ops()
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    res = _rand((m, n), dtype, 1.0, 4)
    b2 = _rand((-(-m // 500), n), torch.float32, 1.0, 5)
    ref = x.float() @ w.float().t() + b
    cases = {"plain": ({}, ref), "stats": ({"stats": True}, ref), "residual": ({"residual": res}, ref + res.float()),
             "bias2": ({"bias2": b2, "rows_per_bias2": 500}, ref + b2.repeat_interleave(500, dim=0)[:m]),
             "silu": ({"act": ops.ACT_SILU, "stats": True}, F.silu(ref))}
    for name, (kw, r) in cases.items():
        out, widths = _launched_widths(ops, lambda: ops.linear(x, w, b, block_n=256, **kw))
        assert widths == [_fitted(ops, n, -(-m // 128))], (name, widths)
        check(f"linear {name} {m}x{k}x{n} {dtype}", out, r, *TOL[dtype])
        _same(f"linear {name} {m}x{k}x{n}", out, ops.linear(x, w, b, block_n=64, **kw))


@pytest.mark.parametrize("dtype", DTYPES)
def test_conv3x3_two_sources_odd_size(dtype):
    """15 x 17 pixels: the pixel boxes overhang both edges, so the masked rows of the 16-byte stores are exercised."""
    ops = _ops()
    nb, h, wd, c1, c2, cout = 40, 15, 17, 128, 64, 320
    x1 = _rand((nb, h, wd, c1), dtype, 1.0, 1)
    x2 = _rand((nb, h, wd, c2), dtype, 1.0, 2)
    wt = _rand((cout, c1 + c2, 3, 3), dtype, (9 * (c1 + c2)) ** -0.5, 3)
    wk = wt.permute(0, 2, 3, 1).reshape(cout, -1).contiguous()
    b = _rand((cout,), torch.float32, 1.0, 4)
    temb = _rand((nb, cout), torch.float32, 1.0, 5)
    res = _rand((nb * h * wd, cout), dtype, 1.0, 6)
    ref = F.conv2d(torch.cat([x1, x2], dim=-1).float().permute(0, 3, 1, 2), wt.float(), b, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, cout)
    for name, kw, r in (("bias2", {"bias2": temb, "rows_per_bias2": h * wd}, ref + temb.repeat_interleave(h * wd, dim=0)),
                        ("residual", {"residual": res}, ref + res.float()), ("stats", {"stats": True}, ref)):
        out, widths = _launched_widths(ops, lambda: ops.conv3x3(x1, wk, b, x2=x2, **kw))
        assert widths == [_fitted(ops, cout, 160)], widths          # boxes of 32 x 4 pixels: 4 m-tiles per image
        check(f"conv3x3 {name} {dtype}", out, r, *TOL[dtype])
        _same(f"conv3x3 {name}", out, ops.conv3x3(x1, wk, b, x2=x2, block_n=64, **kw))


@pytest.mark.parametrize("dtype", DTYPES)
def test_tconv3_widths(dtype):
    ops = _ops()
    b, t, hw, c = 16, 17, 100, 640           # one partly filled 128-pixel tile per frame: 272 m-tiles
    x = _rand((b * t * hw, c), dtype, 1.0, 1)
    wt = _rand((c, 3 * c), dtype, (3 * c) ** -0.5, 2)
    bias = _rand((c,), torch.float32, 1.0, 3)
    res = _rand((b * t * hw, c), dtype, 1.0, 4)
    x5 = x.float().reshape(b, t, hw, 1, c).permute(0, 4, 1, 2, 3)
    w5 = wt.float().reshape(c, 3, c).permute(0, 2, 1).reshape(c, c, 3, 1, 1)
    ref = F.conv3d(x5, w5, bias, padding=(1, 0, 0)).permute(0, 2, 3, 4, 1).reshape(-1, c) + res.float()
    out, widths = _launched_widths(ops, lambda: ops.tconv3(x, b, t, hw, wt, bias, residual=res))
    assert widths == [_fitted(ops, c, 272)], widths
    check(f"tconv3 {dtype}", out, ref, *TOL[dtype])
    _same("tconv3", out, ops.tconv3(x, b, t, hw, wt, bias, residual=res, block_n=64))


@pytest.mark.parametrize("dtype", DTYPES)
def test_geglu_slab_epilogue(dtype):
    """GEGLU keeps its 256- / 128-column tiles; its outputs take the slab epilogue.  1500 rows: partial last m-tile."""
    ops = _ops()
    m, k, n = 1500, 320, 2560
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 0.5, 3)
    y = x.float() @ w.float().t() + b
    ref = y[:, : n // 2] * F.gelu(y[:, n // 2:])
    out = ops.linear(x, w, b, geglu=True)
    check(f"geglu {dtype}", out, ref, *TOL[dtype])
    assert torch.equal(out, ops.linear(x, w, b, geglu=True, block_n=128))
