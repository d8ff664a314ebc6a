"""CPU: which implicit-GEMM launches take the staged epilogue (TMA-stored output tile, column statistics) and which the host
routes to the per-element epilogue before any launch, as `aab_igemm_emits_colstats` reports it (pure host logic)."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    from animate_anything_b200 import _lib
    return _lib


def _desc(_lib, **kw):
    d = _lib.IgemmDesc()
    d.a = d.b = 1 << 20
    d.out = kw.pop("out", 1 << 20)
    d.kc, d.num_taps, d.n, d.block_n, d.out_scale = 64, 1, 256, 256, 1.0
    d.ld_out = kw.pop("ld_out", 256)
    dims, box = kw.pop("dim_d", (4096, 1, 1, 1)), kw.pop("box", (128, 1, 1, 1))
    for i in range(4):
        d.dim_d[i], d.box[i] = dims[i], box[i]
    d.colstats = 1
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _staged(_lib, **kw):
    return bool(_lib.load().aab_igemm_emits_colstats(C.byref(_desc(_lib, **kw))))


def test_staged_layouts(lib):
    assert _staged(lib)
    assert _staged(lib, ld_out=512)                                            # column slice, 16-byte row pitch
    assert _staged(lib, residual=1 << 21, ld_res=264)                          # residual with its own pitch
    assert _staged(lib, bias2=1 << 22, rows_per_bias2=500, ld_bias2=256)       # a tile spans at most two samples
    assert _staged(lib, bias2=1 << 22, rows_per_bias2=128, ld_bias2=256)
    # conv3x3-like tiles (64 x 2 pixels of a 64 x 64 frame): a tile spans 64 + 64 rows of one frame
    assert _staged(lib, dim_d=(64, 64, 32, 1), box=(64, 2, 1, 1), bias2=1 << 22, rows_per_bias2=16 * 4096, ld_bias2=256)


def test_layouts_routed_to_direct(lib):
    assert not _staged(lib, ld_out=260)                                        # row pitch not a multiple of 16 bytes
    assert not _staged(lib, out=(1 << 20) + 8)                                 # base not 16-byte aligned
    assert not _staged(lib, residual=1 << 21, ld_res=260)
    assert not _staged(lib, residual=(1 << 21) + 4, ld_res=256)
    assert not _staged(lib, bias2=1 << 22, rows_per_bias2=100, ld_bias2=256)   # three samples in one tile
    assert not _staged(lib, dim_d=(64, 64, 32, 1), box=(64, 2, 1, 1), bias2=1 << 22, rows_per_bias2=64, ld_bias2=256)
    assert not _staged(lib, ld_out=1 << 28, dim_d=(1 << 12, 1, 1, 1))          # a stride of 2^40 bytes or more
    assert not _staged(lib, dim_d=(1 << 16, 1 << 15, 1, 1))                    # 2^31 rows
    assert not _staged(lib, n=250)                                             # n_out not a multiple of 32
