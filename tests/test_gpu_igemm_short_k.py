"""Two CTAs per SM for the short-K 1-tap launches of the implicit GEMM (`ops.pick_two_cta`): every output and
column-statistics table is bit-identical to the same launch forced onto the one-CTA path (same K order, same epilogue
arithmetic), and within the 16-bit rounding of the fp32 torch reference."""
import pytest
import torch

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


def _launches(ops, fn):
    """Run fn() and return (result, [(tile width, two CTAs per SM)] of the implicit-GEMM launches it made)."""
    ops.IGEMM_PROFILE = []
    try:
        out = fn()
        launched = [(p["block_n"], p["two_cta"]) for p in ops.IGEMM_PROFILE]
    finally:
        ops.IGEMM_PROFILE = None
    return out, launched


def _same(name, two, one):
    assert torch.equal(two, one), f"{name}: two CTAs per SM differ from one"
    s2, s1 = getattr(two, "_aab_stats", None), getattr(one, "_aab_stats", None)
    assert (s2 is None) == (s1 is None), name
    if s2 is not None:
        assert torch.equal(s2, s1), f"{name}: column statistics differ"


# 139264 / 34816 rows = the 64x64 / 32x32 levels of a config-2 forward (2 x 17 frames x 4096 / 1024 pixels); 34048 rows =
# 266 m-tiles, just above the 264 CTAs of two per SM on 132 SMs.  139227 and 34000 rows end in a partial m-tile (no column
# statistics: `linear` asks for them only when every m-tile is whole).  K = 64 / 320 / 640, N = 320 ... 1920.
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m,k,n", [(139264, 320, 320), (139227, 320, 320), (139264, 320, 960), (34048, 320, 1280),
                                   (34000, 64, 320), (34816, 640, 640), (34000, 640, 640), (34816, 640, 1920)])
def test_linear_two_cta(dtype, m, k, n):
    ops = _ops()
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    res = _rand((m, n), dtype, 1.0, 4)
    ref = x.float() @ w.float().t()
    cases = {"plain": ({"bias": b}, ref + b), "no bias": ({}, ref),
             "residual": ({"bias": b, "residual": res}, ref + b + res.float()),
             "residual+stats": ({"bias": b, "residual": res, "stats": True}, ref + b + res.float()),
             "stats": ({"bias": b, "stats": True}, ref + b)}
    m_tiles = -(-m // 128)
    assert ops.pick_two_cta(n, m_tiles, k, 1) == 64
    for name, (kw, r) in cases.items():
        kw = dict(kw)
        bias = kw.pop("bias", None)
        out, launched = _launches(ops, lambda: ops.linear(x, w, bias, **kw))
        assert launched == [(64, True)], (name, launched)
        check(f"linear {name} {m}x{k}x{n} {dtype}", out, r, *TOL[dtype])
        if kw.get("stats") and m % 128 == 0:
            st = out._aab_stats
            assert st.shape == (m_tiles, n, 2), name
            o = torch.nn.functional.pad(out.float(), (0, 0, 0, m_tiles * 128 - m)).view(m_tiles, 128, n)
            check(f"colstats sum {name}", st[..., 0], o.sum(1), 1e-4, 1e-2)
            check(f"colstats sumsq {name}", st[..., 1], (o * o).sum(1), 1e-4, 1e-2)
        one, launched1 = _launches(ops, lambda: ops.linear(x, w, bias, ctas_per_sm=1, **kw))
        assert launched1 and not launched1[0][1], launched1
        _same(f"linear {name} {m}x{k}x{n} {dtype}", out, one)
        _same(f"linear {name} {m}x{k}x{n} {dtype} BN 64", out, ops.linear(x, w, bias, block_n=64, ctas_per_sm=1, **kw))


@pytest.mark.parametrize("dtype", DTYPES)
def test_direct_epilogue_two_cta(dtype):
    """fp32 and scaled outputs (per-element stores from the registers) when a caller forces two CTAs per SM."""
    ops = _ops()
    m, k, n = 34000, 320, 330
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 1.0, 3)
    res = _rand((m, n), dtype, 1.0, 4)
    for name, kw in {"fp32": {"out_f32": True}, "scaled residual": {"residual": res, "out_scale": 0.5},
                     "odd n": {}}.items():
        two = ops.linear(x, w, b, block_n=64, ctas_per_sm=2, **kw)
        one = ops.linear(x, w, b, block_n=64, ctas_per_sm=1, **kw)
        assert torch.equal(two, one), name
        ref = x.float() @ w.float().t() + b
        if "residual" in kw:
            ref = (ref + res.float()) * 0.5
        check(f"direct {name} {dtype}", two, ref, *TOL[dtype])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [320, 960, 2560])
def test_geglu_stays_one_cta(dtype, n):
    """GEGLU needs 128-column tiles, whose accumulators do not fit two CTAs per SM: the rule leaves it on the one-CTA
    path, and forcing it is rejected before any launch."""
    ops = _ops()
    m, k = 34000, 320
    x = _rand((m, k), dtype, 1.0, 1)
    w = _rand((n, k), dtype, k ** -0.5, 2)
    b = _rand((n,), torch.float32, 0.5, 3)
    out, launched = _launches(ops, lambda: ops.linear(x, w, b, geglu=True))
    assert len(launched) == 1 and not launched[0][1], launched
    h = x.float() @ w.float().t() + b
    ref = h[:, : n // 2] * torch.nn.functional.gelu(h[:, n // 2:])
    check(f"geglu {m}x{k}x{n} {dtype}", out, ref, *TOL[dtype])
    with pytest.raises(ops._lib.AabError):
        ops.linear(x, w, b, geglu=True, block_n=128, ctas_per_sm=2)


def test_rule_leaves_other_launches_alone():
    ops = _ops()
    x = _rand((34816, 1280), torch.bfloat16, 1.0, 1)
    w = _rand((320, 1280), torch.bfloat16, 1280 ** -0.5, 2)
    _, launched = _launches(ops, lambda: ops.linear(x, w, None))          # K = 1280
    assert not launched[0][1], launched
    x = _rand((16000, 320), torch.bfloat16, 1.0, 1)
    w = _rand((320, 320), torch.bfloat16, 320 ** -0.5, 2)
    _, launched = _launches(ops, lambda: ops.linear(x, w, None))          # 125 m-tiles: fewer than 2 x 132
    assert not launched[0][1], launched
