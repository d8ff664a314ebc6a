"""Tensor-level wrappers over the C-ABI (`_lib.call`).  Activations are channels-last 16-bit torch tensors; torch only
provides memory and the current stream.  Every function here launches hand-written sm_90a kernels — nothing falls back
to torch compute.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import (ACT_GELU, ACT_NONE, ACT_QUICK_GELU, ACT_SILU, F_BF16, F_DIRECT, F_GEGLU, F_OUT_F32, F_SCALE_ACC, F_TWO_CTA,
                   IgemmDesc)

NUM_SMS = 132           # H100 SXM
IGEMM_PROFILE = None     # bench.py sets this to a list to time every implicit-GEMM launch with CUDA events
KERNEL_PROFILE = None    # same for the other kernels: list of {"name", "bytes" (algorithmic HBM bytes), "flops", "ev"}


def _profiled(name, nbytes, flops, fn, shape=None):
    """Run `fn` (one C-ABI call); when KERNEL_PROFILE is a list, bracket it with CUDA events on the launch stream."""
    if KERNEL_PROFILE is None:
        return fn()
    ev0 = torch.cuda.Event(enable_timing=True)
    ev1 = torch.cuda.Event(enable_timing=True)
    ev0.record()
    r = fn()
    ev1.record()
    KERNEL_PROFILE.append({"name": name, "bytes": float(nbytes), "flops": float(flops), "ev": (ev0, ev1), "shape": shape})
    return r


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _is_bf16(t: torch.Tensor) -> int:
    if t.dtype == torch.bfloat16:
        return 1
    if t.dtype == torch.float16:
        return 0
    raise TypeError(f"16-bit activations required, got {t.dtype}")


def _np2(x: int) -> int:
    return 1 << max(0, (int(x) - 1).bit_length())


def pick_box(dims: Sequence[int], fixed_one: Sequence[int] = ()) -> list:
    """Pixels-per-tile along each (innermost-first) output dim; powers of two with product 128."""
    box = [1, 1, 1, 1]
    rem = 128
    for i, d in enumerate(dims):
        if i in fixed_one:
            continue
        b = min(rem, _np2(d))
        box[i] = b
        rem //= b
        if rem == 1:
            break
    if rem > 1:
        for i in range(4):
            if i not in fixed_one:
                box[i] *= rem
                break
    return box


def _tiles_cover_rows_in_order(dim_d, box) -> bool:
    """True when m-tile i of the kernel's tile order holds exactly the output rows [128 i, 128 i + 128): every dim below
    the first partially-boxed one is boxed whole, every dim above it has box 1, and the boxes divide the dims."""
    i = 0
    while i < 4 and box[i] == dim_d[i]:
        i += 1
    if i < 4:
        if dim_d[i] % box[i]:
            return False
        i += 1
    return all(box[j] == 1 for j in range(i, 4))


def pick_block_n(n_out: int, m_tiles: int, geglu: bool = False, k_total: int = 1 << 30) -> int:
    """Widest tile allowed (GEMM columns: 32 / 64 / 128 / 256).  Wide tiles win wherever the main loop dominates: every
    k-block loads the same 16 KiB of activations whatever the width, so a wide tile reads A once for more columns.  A ragged
    last N tile costs no traffic (TMA zero-fill beyond N) but issues every MMA of its dead columns, so `igemm` narrows a
    256-column answer to the width that fits N and the wave count (`fit_block_n`)."""
    if geglu:
        return 256 if n_out > 64 else 128
    if m_tiles <= 2:
        return 64           # weight-streaming (GEMV-like: text K/V, time embedding): spread the weight rows over many CTAs
    if n_out <= 64:
        # a 64-column output on a 256-column tile computes and stages mostly zero-filled weight rows; UNet384's 64-channel
        # levels (1-4 M rows) are HBM / latency bound and want the narrow tile.  No shape of the SD UNet / VAE / SVD / CLIP
        # paths has N <= 64.
        return 64
    if k_total <= 384 and n_out <= 640:
        # epilogue/HBM-bound (tiny K): more tiles than SMs keep every SM busy
        return 128 if m_tiles * -(-n_out // 128) >= NUM_SMS else 64
    return 256


def fit_block_n(n_out: int, m_tiles: int, sms: int = NUM_SMS) -> int:
    """Width actually launched where up to 256 columns are allowed.  All tiles of a launch have one width w and the launch
    takes ceil(tiles / SMs) waves of w columns each, dead columns of a ragged last tile included: minimise waves * w over
    128 / 160 / 192 / 256.  Costs within 5 % of the minimum tie and the widest wins a tie (fewer A re-reads per flop).
    N <= 256 is one n-tile today and stays so.  The K order of an output element does not depend on the width, so
    results are bit-identical whichever is chosen."""
    if n_out <= 256:
        return 256
    cost = {w: -(-(m_tiles * -(-n_out // w)) // sms) * w for w in (128, 160, 192, 256)}
    best = min(cost.values())
    return max(w for w, c in cost.items() if c <= 1.05 * best)


def pick_two_cta(n_out: int, m_tiles: int, k_total: int, taps: int, geglu: bool = False) -> int:
    """Tile width of the two-CTAs-per-SM configuration for this launch, or 0 for the one-CTA path (`pick_block_n`).
    With K <= 640 a tile is at most ten k-blocks of MMAs; with one CTA per SM its epilogue (bias, residual, stores) and
    the ring refill for the next tile run with the tensor cores idle, and a second resident CTA fills that gap.  64-column
    tiles only: the one width whose accumulators fit the 80 registers of two 384-thread CTAs (GEGLU needs 128).  Only with
    at least one m-tile per resident CTA.  On an H100 at 700 W (tools/igemm_short_k.py, graph-replayed) every 1-tap
    transformer linear of config 2 at K = 320 and 640 gains 12 - 43 % against the one-CTA widths (DESIGN.md section 6)."""
    if geglu or taps != 1 or k_total > 640 or m_tiles < 2 * NUM_SMS or n_out < 320:
        return 0
    return 64


def _fix_strides(dims, strides):
    """TMA wants non-zero, 16-byte-multiple strides even for extent-1 dims."""
    st = list(strides)
    for i in range(1, 5):
        if st[i] == 0:
            st[i] = st[i - 1] * max(1, dims[i - 1])
    return st


def igemm(a: torch.Tensor, a_dims, a_strides, w: torch.Tensor, n: int, kc: int, dim_d, box, taps,
          out: Optional[torch.Tensor] = None, ld_out: Optional[int] = None, *, bias=None, bias2=None, rows_per_bias2=1,
          residual=None, ld_res=None, act=ACT_NONE, out_scale=1.0, geglu=False, out_f32=False, a2=None, a2_dims=None,
          a2_strides=None, kc1=0, ld_b=None, b_batch=0, b_batch_stride=0, b_batch_dim=-1, block_n=None, direct=False,
          out_rows=None, scale_acc=False, stats=False, ctas_per_sm=None):
    """Generic launch of the implicit-GEMM kernel. `taps` is a list of 5-int offsets (channel, pix0..pix3).
    `block_n` / `ctas_per_sm` (1, or 2 with `block_n=64`) override the tile width and the CTAs per SM that `pick_two_cta`
    / `pick_block_n` choose from the shape; results are bit-identical whichever runs.
    `stats=True`: the output feeds a GroupNorm -- have the epilogue also write per-(128-row tile, column) sums / sums of
    squares of the rounded outputs (`out._aab_stats`, [m_tiles, n, 2] fp32) so that `groupnorm` can skip its statistics read.
    Silently not produced when the launch takes an epilogue that cannot (the consumer then runs the two-pass GroupNorm)."""
    bf = _is_bf16(a)
    n_out = n // 2 if geglu else n
    rows = 1
    for d in dim_d:
        rows *= d
    if out is None:
        out = torch.empty((rows if out_rows is None else out_rows, n_out), device=a.device,
                          dtype=torch.float32 if out_f32 else a.dtype)
    if ld_out is None:
        ld_out = out.stride(-2) if out.dim() >= 2 else n_out
    d = IgemmDesc()
    d.a = a.data_ptr()
    a_strides = _fix_strides(a_dims, a_strides)
    for i in range(5):
        d.a_dims[i] = a_dims[i]
        d.a_strides[i] = a_strides[i]
    if a2 is not None:
        d.a2 = a2.data_ptr()
        a2_strides = _fix_strides(a2_dims, a2_strides)
        for i in range(5):
            d.a2_dims[i] = a2_dims[i]
            d.a2_strides[i] = a2_strides[i]
        d.kc1 = kc1
    else:
        d.a2 = None
    d.kc = kc
    d.num_taps = len(taps)
    for t, off in enumerate(taps):
        for j in range(5):
            d.tap_off[t][j] = off[j]
    d.b = w.data_ptr()
    d.ld_b = ld_b if ld_b is not None else w.stride(-2)
    d.b_batch = b_batch
    d.b_batch_stride = b_batch_stride
    d.b_batch_dim = b_batch_dim
    d.n = n
    m_tiles = 1
    for i in range(4):
        d.dim_d[i] = dim_d[i]
        d.box[i] = box[i]
        m_tiles *= -(-dim_d[i] // box[i])
    d.out = out.data_ptr()
    d.ld_out = ld_out
    d.bias = None if bias is None else bias.data_ptr()
    if bias is not None:
        assert bias.dtype == torch.float32
    if bias2 is not None:
        assert bias2.dtype == torch.float32
        d.bias2 = bias2.data_ptr()
        d.rows_per_bias2 = rows_per_bias2
        d.ld_bias2 = bias2.stride(0)
    else:
        d.bias2 = None
        d.rows_per_bias2 = 1
    if residual is not None:
        d.residual = residual.data_ptr()
        d.ld_res = ld_res if ld_res is not None else residual.stride(-2)
    else:
        d.residual = None
    d.out_scale = out_scale
    d.act = act
    flags = ((F_BF16 if bf else 0) | (F_GEGLU if geglu else 0) | (F_OUT_F32 if out_f32 else 0) | (F_DIRECT if direct else 0) |
             (F_SCALE_ACC if scale_acc else 0))
    if block_n is None and ctas_per_sm is None:
        block_n = pick_two_cta(n_out, m_tiles, kc * len(taps), len(taps), geglu) or None
        ctas_per_sm = 2 if block_n else 1
    if ctas_per_sm == 2:
        flags |= F_TWO_CTA
    if block_n is None:
        if n_out < 64 and not geglu:
            # 32-column tiles only have the direct-store epilogue; an output that qualifies for the staged epilogue (and
            # its column statistics) takes a 64-column tile whose upper half is a ragged, zero-filled N remainder instead
            staged_ok = n_out % 32 == 0 and not out_f32 and not direct and not scale_acc and ld_out % 8 == 0
            block_n = 64 if (n_out > 32 or staged_ok) else 32
        else:
            block_n = pick_block_n(n_out, m_tiles, geglu, kc * len(taps))
    if block_n == 256 and not geglu:
        block_n = fit_block_n(n_out, m_tiles, _lib.load().aab_num_sms())
    d.flags = flags
    d.block_n = block_n
    cstats = None
    if stats and not geglu and _tiles_cover_rows_in_order(dim_d, box):
        d.colstats = 1          # placeholder so that the C-side predicate sees "requested"
        if _lib.load().aab_igemm_emits_colstats(C.byref(d)):
            cstats = torch.empty((m_tiles, n_out, 2), device=a.device, dtype=torch.float32)
            d.colstats = cstats.data_ptr()
        else:
            d.colstats = None
    if cstats is not None:
        out._aab_stats = cstats
    if IGEMM_PROFILE is not None:
        ev0 = torch.cuda.Event(enable_timing=True)
        ev1 = torch.cuda.Event(enable_timing=True)
        ev0.record()
        _lib.call("aab_igemm", C.byref(d), _stream())
        ev1.record()
        IGEMM_PROFILE.append({"rows": rows, "n": n, "k": kc * len(taps), "taps": len(taps), "block_n": block_n,
                              "two_cta": bool(flags & F_TWO_CTA), "geglu": geglu,
                              "residual": residual is not None,
                              "flops": 2.0 * rows * n * kc * len(taps), "ev": (ev0, ev1)})
    else:
        _lib.call("aab_igemm", C.byref(d), _stream())
    return out


_NO_TAP = [[0, 0, 0, 0, 0]]
TAPS_3X3 = [[0, s - 1, r - 1, 0, 0] for r in range(3) for s in range(3)]
TAPS_T3 = [[0, 0, dt - 1, 0, 0] for dt in range(3)]


def linear(x: torch.Tensor, w: torch.Tensor, bias=None, **kw) -> torch.Tensor:
    """x [M, K] (row stride arbitrary, multiple of 8) @ w[N, K]^T."""
    m, k = x.shape
    n = w.shape[0]
    return igemm(x, (k, m, 1, 1, 1), (1, x.stride(0), 0, 0, 0), w, n, k, (m, 1, 1, 1), (128, 1, 1, 1), _NO_TAP,
                 bias=bias, **kw)


def conv3x3(x: torch.Tensor, w: torch.Tensor, bias=None, x2: Optional[torch.Tensor] = None, **kw) -> torch.Tensor:
    """x [N, H, W, C] channels-last (optionally virtually concatenated with x2 on channels), w [Cout, 9*(C+C2)]
    tap-major (r, s, c).  stride 1, zero padding 1.  Returns [N*H*W, Cout]."""
    nb, h, wd, c = x.shape
    dims = (c, wd, h, nb, 1)
    strides = (1, c, wd * c, h * wd * c, nb * h * wd * c)
    dim_d = (wd, h, nb, 1)
    box = pick_box(dim_d)
    if x2 is not None:
        c2 = x2.shape[-1]
        return igemm(x, dims, strides, w, w.shape[0], c + c2, dim_d, box, TAPS_3X3, bias=bias, a2=x2,
                     a2_dims=(c2, wd, h, nb, 1), a2_strides=(1, c2, wd * c2, h * wd * c2, nb * h * wd * c2), kc1=c, **kw)
    return igemm(x, dims, strides, w, w.shape[0], c, dim_d, box, TAPS_3X3, bias=bias, **kw)


def conv1x1_cat(x: torch.Tensor, x2: Optional[torch.Tensor], w: torch.Tensor, bias=None, **kw) -> torch.Tensor:
    """1x1 conv / linear over the virtual channel concat of x [M, C1] and x2 [M, C2]."""
    m, c = x.shape
    if x2 is None:
        return linear(x, w, bias, **kw)
    c2 = x2.shape[1]
    return igemm(x, (c, m, 1, 1, 1), (1, x.stride(0), 0, 0, 0), w, w.shape[0], c + c2, (m, 1, 1, 1), (128, 1, 1, 1),
                 _NO_TAP, bias=bias, a2=x2, a2_dims=(c2, m, 1, 1, 1), a2_strides=(1, x2.stride(0), 0, 0, 0), kc1=c, **kw)


def conv3x3_stride2(x: torch.Tensor, w: torch.Tensor, bias=None, pad_mode: str = "sym", **kw) -> torch.Tensor:
    """3x3 stride-2 conv on x [N, H, W, C] (H, W even) through a space-to-depth view (no gather kernel).
    pad_mode "sym": padding 1 (UNet Downsample2D); "br": F.pad(0,1,0,1) + padding 0 (VAE encoder Downsample2D)."""
    nb, h, wd, c = x.shape
    assert h % 2 == 0 and wd % 2 == 0 and c % 64 == 0
    h2, w2 = h // 2, wd // 2
    dims = (2 * c, w2, 2, h2, nb)
    strides = (1, 2 * c, wd * c, 2 * wd * c, h * wd * c)
    dim_d = (w2, 1, h2, nb)
    box = pick_box(dim_d, fixed_one=(1,))
    if pad_mode == "sym":
        m = {0: (1, -1), 1: (0, 0), 2: (1, 0)}      # kernel index -> (parity, coarse offset)
    else:
        m = {0: (0, 0), 1: (1, 0), 2: (0, 1)}
    taps = []
    for r in range(3):
        hp, dh = m[r]
        for s in range(3):
            wp, dw = m[s]
            taps.append([wp * c, dw, hp, dh, 0])
    return igemm(x, dims, strides, w, w.shape[0], c, dim_d, box, taps, bias=bias, **kw)


def tconv3(x: torch.Tensor, b: int, t: int, hw: int, w: torch.Tensor, bias=None, **kw) -> torch.Tensor:
    """Conv3d kernel (3,1,1), padding (1,0,0) on x [B*T*HW, C] in (b, t, hw) row order; w [Cout, 3*C] tap-major."""
    c = x.shape[-1]
    dims = (c, hw, t, b, 1)
    strides = (1, c, hw * c, t * hw * c, b * t * hw * c)
    dim_d = (hw, t, b, 1)
    box = pick_box(dim_d)
    return igemm(x, dims, strides, w, w.shape[0], c, dim_d, box, TAPS_T3, bias=bias, **kw)


# ---------------------------------------------------------------------------------------------- attention
def flash_attn_d64(q: torch.Tensor, q_col0: int, kv: torch.Tensor, k_col0: int, v_col0: int, nb: int, lq: int, lk: int,
                   heads: int, kv_batch_div: int = 1, out: Optional[torch.Tensor] = None, causal: bool = False,
                   scale: Optional[float] = None) -> torch.Tensor:
    """q: [nb*lq, q_cols]; kv: [nb_kv*lk, kv_cols]; head h uses columns col0 + 64*h.  Returns [nb*lq, heads*64].
    `causal` (lq == lk <= 128): key j is visible to query i iff j <= i (CLIP text tower).
    `scale`: softmax scale, default 1/sqrt(64); heads narrower than 64 are run zero-padded to 64 columns with their own
    1/sqrt(head_dim) (UNet384's head dim 8: zero columns add exact zeros to Q.K^T and produce zero output columns)."""
    bf = _is_bf16(q) | (2 if causal else 0)
    if out is None:
        out = torch.empty((nb * lq, heads * 64), device=q.device, dtype=q.dtype)
    nb_kv = kv.shape[0] // lk
    _profiled("flash_attn_d64", 2.0 * 64 * heads * (2 * nb * lq + 2 * nb_kv * lk), 4.0 * nb * heads * lq * lk * 64,
              lambda: _lib.call("aab_flash_attn_d64", _ptr(q), q.stride(0), lq * q.stride(0), q.shape[1], q_col0,
                                _ptr(kv), kv.stride(0), lk * kv.stride(0), kv.shape[1], k_col0, v_col0,
                                _ptr(out), out.stride(0), lq * out.stride(0), 0, nb, nb_kv, kv_batch_div, heads, lq, lk,
                                1.0 / math.sqrt(64.0) if scale is None else float(scale), bf, _stream()),
              shape=(nb, heads, lq, lk))
    return out


def flash_attn_d80(q: torch.Tensor, q_col0: int, kv: torch.Tensor, k_col0: int, v_col0: int, nb: int, lq: int, lk: int,
                   heads: int, kv_batch_div: int = 1, out: Optional[torch.Tensor] = None,
                   scale: Optional[float] = None) -> torch.Tensor:
    """Bidirectional attention with head dim 80 (CLIP ViT-H/14 image tower).  q: [nb*lq, q_cols]; kv: [nb_kv*lk, kv_cols];
    head h uses columns col0 + 80*h.  Returns [nb*lq, heads*80].  `scale`: softmax scale, default 1/sqrt(80)."""
    bf = _is_bf16(q)
    if out is None:
        out = torch.empty((nb * lq, heads * 80), device=q.device, dtype=q.dtype)
    nb_kv = kv.shape[0] // lk
    _profiled("flash_attn_d80", 2.0 * 80 * heads * (2 * nb * lq + 2 * nb_kv * lk), 4.0 * nb * heads * lq * lk * 80,
              lambda: _lib.call("aab_flash_attn_d80", _ptr(q), q.stride(0), lq * q.stride(0), q.shape[1], q_col0,
                                _ptr(kv), kv.stride(0), lk * kv.stride(0), kv.shape[1], k_col0, v_col0,
                                _ptr(out), out.stride(0), lq * out.stride(0), 0, nb, nb_kv, kv_batch_div, heads, lq, lk,
                                1.0 / math.sqrt(80.0) if scale is None else float(scale), bf, _stream()),
              shape=(nb, heads, lq, lk))
    return out


def single_head_attention(qkv: torch.Tensor, n: int, l: int, c: int) -> torch.Tensor:
    """softmax(Q K^T / sqrt(c)) V per frame, one head of width c (AutoencoderKL mid-block attention, upcast_softmax).
    qkv: [n*l, 3c] with columns (q, k, v).  Returns [n*l, c].  S and O are batched implicit GEMMs along the frames, the
    softmax runs on fp32 scores; the K of the P.V GEMM is l rounded up to a multiple of 8, padded with zero probabilities
    and zero V columns."""
    lp = (l + 7) // 8 * 8
    s = igemm(qkv, (c, l, n, 1, 1), (1, 3 * c, l * 3 * c, 0, 0), qkv[:, c:2 * c], l, c, (l, n, 1, 1), (128, 1, 1, 1),
              _NO_TAP, ld_b=3 * c, b_batch=n, b_batch_stride=l * 3 * c, b_batch_dim=1, out_f32=True,
              out_scale=1.0 / math.sqrt(c))
    pr = softmax_rows(s, qkv.dtype, pad_to=lp)                         # [n*l, lp]
    vt = transpose_batched(qkv, 2 * c, n, l, c, ld=lp)                 # [n, c, lp]
    return igemm(pr, (lp, l, n, 1, 1), (1, lp, l * lp, 0, 0), vt, c, lp, (l, n, 1, 1), (128, 1, 1, 1), _NO_TAP, ld_b=lp,
                 b_batch=n, b_batch_stride=c * lp, b_batch_dim=1)


_SRC_TYPES = {torch.uint8: 0, torch.float32: 1, torch.float16: 2, torch.bfloat16: 3}


def clip_image_prep(src: torch.Tensor, dtype, out_size: int, patch: int, k_pad: int, taps_y: Optional[torch.Tensor] = None,
                    taps_x: Optional[torch.Tensor] = None, mean_std: Optional[torch.Tensor] = None) -> torch.Tensor:
    """CLIP image preprocessing + patchify (`aab_clip_image_prep`).  `src`: uint8 images [B, H, W, 3] (full preprocessing:
    blur taps and mean/std as fp32 device tensors) or CLIP pixel values [B, 3, S, S] of any float dtype (rounding only).
    Returns the patch-embedding GEMM operand [B * (1 + (S/patch)^2), k_pad] in `dtype`: row 0 of each image is the zero
    class slot, then the patches, columns >= 3 patch^2 zero."""
    if src.dtype not in _SRC_TYPES:
        raise TypeError(f"image source must be uint8 or float, got {src.dtype}")
    if src.dtype == torch.uint8:
        b, h, w, c = src.shape
        sb, sy, sx, sc = src.stride()
        assert taps_y is not None and taps_x is not None and mean_std is not None
        for t in (taps_y, taps_x, mean_std):
            assert t.dtype == torch.float32 and t.is_contiguous() and t.device == src.device
    else:
        b, c, h, w = src.shape
        sb, sc, sy, sx = src.stride()
    if c != 3:
        raise ValueError(f"CLIP images have 3 channels, got {c}")
    grid = out_size // patch
    out = torch.empty((b * (1 + grid * grid), k_pad), device=src.device, dtype=dtype)
    _lib.call("aab_clip_image_prep", _ptr(src), _SRC_TYPES[src.dtype], sb, sc, sy, sx, b, h, w, _ptr(taps_y),
              0 if taps_y is None else taps_y.numel(), _ptr(taps_x), 0 if taps_x is None else taps_x.numel(), _ptr(mean_std),
              out_size, patch, _ptr(out), out.stride(0), 1 if dtype == torch.bfloat16 else 0, _stream())
    return out


def _temporal_attn(qkv: torch.Tensor, b: int, t: int, hw: int, heads: int, q_col0: int, k_col0: int, v_col0: int,
                   long_clip: bool):
    bf = _is_bf16(qkv) | (2 if long_clip else 0)
    out = torch.empty((qkv.shape[0], heads * 64), device=qkv.device, dtype=qkv.dtype)
    rows = qkv.shape[0]
    _profiled("temporal_attn_d64", 2.0 * rows * heads * 64 * 4, 4.0 * b * hw * heads * t * t * 64,
              lambda: _lib.call("aab_temporal_attn_d64", _ptr(qkv), qkv.stride(0), q_col0, k_col0, v_col0, _ptr(out),
                                out.stride(0), b, t, hw, heads, 1.0 / math.sqrt(64.0), bf, _stream()),
              shape=(b, t, hw, heads))
    return out


def temporal_attn_d64(qkv: torch.Tensor, b: int, t: int, hw: int, heads: int, q_col0: int, k_col0: int, v_col0: int):
    return _temporal_attn(qkv, b, t, hw, heads, q_col0, k_col0, v_col0, long_clip=False)


# The long-clip kernel keeps a 16-query tile's whole score row (up to 128 keys) in registers; longer clips would need an
# online softmax over key blocks.
TEMPORAL_MAX_FRAMES = 128


def temporal_attn_long(qkv: torch.Tensor, b: int, t: int, hw: int, heads: int, q_col0: int, k_col0: int, v_col0: int):
    """`temporal_attn_d64` on the long-clip kernel (bit 1 of `is_bf16`): t in 1..TEMPORAL_MAX_FRAMES, same layout."""
    return _temporal_attn(qkv, b, t, hw, heads, q_col0, k_col0, v_col0, long_clip=True)


def temporal_attn(qkv: torch.Tensor, b: int, t: int, hw: int, heads: int, q_col0: int, k_col0: int, v_col0: int):
    """Self-attention over the t frames of every (b, pixel, head), kernel chosen by t: up to 32 frames the v2 kernel
    (`temporal_attn_d64`, unchanged results), 33..TEMPORAL_MAX_FRAMES the long-clip kernel."""
    if t <= 32:
        return temporal_attn_d64(qkv, b, t, hw, heads, q_col0, k_col0, v_col0)
    if t <= TEMPORAL_MAX_FRAMES:
        return temporal_attn_long(qkv, b, t, hw, heads, q_col0, k_col0, v_col0)
    raise NotImplementedError(f"temporal attention handles up to {TEMPORAL_MAX_FRAMES} frames, got {t}")


# ---------------------------------------------------------------------------------------------- norms
# Samples (frames, for the spatial norms) per GroupNorm launch: the per-sample tickets of `aab_groupnorm` (csrc/norm.cu)
GN_MAX_SAMPLES = 4096
_gn_ws = {}


def _gn_workspace(device, nbytes):
    """Zero-initialised (tickets!) workspace per (device, stream); the kernel leaves the tickets at zero."""
    key = (device, torch.cuda.current_stream().cuda_stream)
    buf = _gn_ws.get(key)
    if buf is None or buf.numel() < nbytes:
        # 8 MiB covers every extent of the path (largest: VAE decoder, 8 frames x 1024 chunks = 4.2 MiB), so the buffer is
        # never re-grown later -- in particular not in the middle of a CUDA-graph capture, where the old block could be
        # handed to another tensor of the same capture while earlier captured kernels still point at it
        buf = torch.zeros(max(int(nbytes), 8 << 20), device=device, dtype=torch.uint8)
        _gn_ws[key] = buf
    return buf


def groupnorm(x: torch.Tensor, samples: int, rows: int, gamma: torch.Tensor, beta: torch.Tensor, eps: float,
              silu: bool, groups: int = 32, x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [samples*rows, C] (+ optional x2 [.., C2] virtual concat).  Statistics per (sample, group) over rows x C/groups."""
    bf = _is_bf16(x)
    c1 = x.shape[1]
    c2 = 0 if x2 is None else x2.shape[1]
    y = torch.empty((x.shape[0], c1 + c2), device=x.device, dtype=x.dtype)
    need = _lib.load().aab_groupnorm_workspace_bytes(samples, rows, c1 + c2, groups)
    if need < 0:
        raise _lib.AabError("aab_groupnorm: unsupported channel count")
    ws = _gn_workspace(x.device, need)
    st1 = getattr(x, "_aab_stats", None)
    st2 = None if x2 is None else getattr(x2, "_aab_stats", None)
    if st1 is not None and rows % 128 == 0 and (x2 is None or st2 is not None):
        # statistics from the producing GEMMs' epilogues: finalize (tiny) + apply; bytes = one read + one write as before
        assert st1.shape[0] * 128 == x.shape[0] and st1.shape[1] == c1
        _profiled("groupnorm", 2.0 * 2 * x.shape[0] * (c1 + c2), 0.0,
                  lambda: _lib.call("aab_groupnorm_colstats", _ptr(x), x.stride(0), c1, _ptr(st1), _ptr(x2),
                                    0 if x2 is None else x2.stride(0), c2, _ptr(st2), samples, rows, groups, _ptr(gamma),
                                    _ptr(beta), eps, int(silu), _ptr(y), y.stride(0), _ptr(ws), bf, _stream()),
                  shape=(samples, rows, c1 + c2, int(silu), "colstats"))
        return y
    # algorithmic bytes (SURVEY 8d): one read + one write of the activation
    _profiled("groupnorm", 2.0 * 2 * x.shape[0] * (c1 + c2), 0.0,
              lambda: _lib.call("aab_groupnorm", _ptr(x), x.stride(0), c1, _ptr(x2), 0 if x2 is None else x2.stride(0), c2,
                                samples, rows, groups, _ptr(gamma), _ptr(beta), eps, int(silu), _ptr(y), y.stride(0),
                                _ptr(ws), bf, _stream()), shape=(samples, rows, c1 + c2, int(silu)))
    return y


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    bf = _is_bf16(x)
    y = torch.empty_like(x)
    _profiled("layernorm", 2.0 * 2 * x.shape[0] * x.shape[1], 0.0,
              lambda: _lib.call("aab_layernorm", _ptr(x), x.stride(0), _ptr(y), y.stride(0), _ptr(gamma), _ptr(beta),
                                x.shape[0], x.shape[1], eps, bf, _stream()), shape=tuple(x.shape))
    return y


def softmax_rows(s: torch.Tensor, dtype, pad_to: Optional[int] = None) -> torch.Tensor:
    """fp32 scores [rows, L] -> 16-bit probabilities [rows, pad_to or L]; columns beyond L are zeros (K padding)."""
    p = torch.empty((s.shape[0], pad_to or s.shape[1]), device=s.device, dtype=dtype)
    _lib.call("aab_softmax_rows", _ptr(s), s.stride(0), _ptr(p), p.stride(0), s.shape[0], s.shape[1],
              1 if dtype == torch.bfloat16 else 0, _stream())
    return p


# ---------------------------------------------------------------------------------------------- elementwise
def _strides5(t: torch.Tensor):
    arr = (C.c_long * 5)(*t.stride())
    return arr


def unet_in_assemble(sample, cond, mask, t_frames) -> torch.Tensor:
    """sample [B,4,F,h,w], cond [B,4,1,h,w], mask [Bm,1,1,h,w] or None -> [B, T, h, w, 8]."""
    bf = _is_bf16(sample)
    b, _, f, h, w = sample.shape
    out = torch.empty((b, f + 1, h, w, 8), device=sample.device, dtype=sample.dtype)
    ms = _strides5(mask) if mask is not None else None
    _lib.call("aab_unet_in_assemble", _ptr(sample), _strides5(sample), _ptr(cond), _strides5(cond), _ptr(mask), ms,
              0 if mask is None else mask.shape[0], _ptr(out), b, f + 1, h, w, bf, _stream())
    return out


def unet_out_finalize(y: torch.Tensor, b, t, h, w, dtype) -> torch.Tensor:
    out = torch.empty((b, 4, t - 1, h, w), device=y.device, dtype=dtype)
    _lib.call("aab_unet_out_finalize", _ptr(y), y.stride(0), _ptr(out), b, t, h, w, 1 if dtype == torch.bfloat16 else 0,
              _stream())
    return out


def timestep_embed(t: torch.Tensor, b: int, dim: int, dtype) -> torch.Tensor:
    assert t.dtype == torch.float32 and t.is_cuda
    out = torch.empty((b, dim), device=t.device, dtype=dtype)
    _lib.call("aab_timestep_embed", _ptr(t), t.numel(), _ptr(out), b, dim, 1 if dtype == torch.bfloat16 else 0, _stream())
    return out


def embed_tokens(ids: torch.Tensor, tok_emb: torch.Tensor, pos_emb: torch.Tensor, seq_len: int) -> torch.Tensor:
    """ids int64 [rows] -> tok_emb[ids] + pos_emb[row % seq_len]  as [rows, C] (CLIPTextEmbeddings)."""
    assert ids.dtype == torch.int64 and ids.is_contiguous() and tok_emb.is_contiguous() and pos_emb.is_contiguous()
    out = torch.empty((ids.numel(), tok_emb.shape[1]), device=tok_emb.device, dtype=tok_emb.dtype)
    _lib.call("aab_embed_tokens", _ptr(ids), _ptr(tok_emb), _ptr(pos_emb), _ptr(out), ids.numel(), seq_len,
              tok_emb.shape[1], tok_emb.shape[0], _is_bf16(tok_emb), _stream())
    return out


def geglu(x: torch.Tensor) -> torch.Tensor:
    nh = x.shape[1] // 2
    out = torch.empty((x.shape[0], nh), device=x.device, dtype=x.dtype)
    _lib.call("aab_geglu", _ptr(x), x.stride(0), _ptr(out), out.stride(0), x.shape[0], nh, _is_bf16(x), _stream())
    return out


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    n, h, w, c = x.shape
    y = torch.empty((n, 2 * h, 2 * w, c), device=x.device, dtype=x.dtype)
    _lib.call("aab_upsample2x", _ptr(x), _ptr(y), n, h, w, c, _stream())
    return y


def upsample_nearest(x: torch.Tensor, oh: int, ow: int) -> torch.Tensor:
    """F.interpolate(size=(oh, ow), mode="nearest") on channels-last [N, H, W, C]."""
    n, h, w, c = x.shape
    y = torch.empty((n, oh, ow, c), device=x.device, dtype=x.dtype)
    _lib.call("aab_upsample_nearest", _ptr(x), _ptr(y), n, h, w, oh, ow, c, _stream())
    return y


def pad_to_even(x: torch.Tensor) -> torch.Tensor:
    """[N, H, W, C] -> zero-padded at the bottom / right to even H, W (no-op when already even)."""
    n, h, w, c = x.shape
    ph, pw = h + (h & 1), w + (w & 1)
    if (ph, pw) == (h, w):
        return x
    y = torch.empty((n, ph, pw, c), device=x.device, dtype=x.dtype)
    _lib.call("aab_pad_br", _ptr(x), _ptr(y), n, h, w, ph, pw, c, _stream())
    return y


def dup_rows(x: torch.Tensor) -> torch.Tensor:
    """[R, C] -> [2R, C] with both halves equal to x (CFG pair sharing its prefix)."""
    assert x.is_contiguous()
    out = torch.empty((2 * x.shape[0],) + tuple(x.shape[1:]), device=x.device, dtype=x.dtype)
    _lib.call("aab_dup_rows", _ptr(x), _ptr(out), x.numel() * x.element_size(), _stream())
    st = getattr(x, "_aab_stats", None)
    if st is not None and x.shape[0] % 128 == 0:
        # the producer's per-tile column statistics travel with the rows (so that the duplicated tensor takes the same
        # GroupNorm path, bit for bit, as a batch that was computed twice)
        st2 = torch.empty((2 * st.shape[0],) + tuple(st.shape[1:]), device=st.device, dtype=st.dtype)
        _lib.call("aab_dup_rows", _ptr(st), _ptr(st2), st.numel() * st.element_size(), _stream())
        out._aab_stats = st2
    return out


def transpose_batched(src: torch.Tensor, col0: int, nb: int, rows: int, cols: int, ld: Optional[int] = None) -> torch.Tensor:
    """src [nb*rows, ld_src] -> dst [nb, cols, ld or rows] taking columns col0..col0+cols; dst columns >= rows are zeros."""
    ld = ld or rows
    dst = torch.empty((nb, cols, ld), device=src.device, dtype=src.dtype)
    base = C.c_void_p(src.data_ptr() + col0 * 2)
    _lib.call("aab_transpose", base, src.stride(0), rows * src.stride(0), _ptr(dst), nb, rows, cols, ld, _stream())
    return dst


def cfg_scheduler_step(eps: torch.Tensor, ldc: int, cfg: bool, guidance: float, x: torch.Tensor, x_out: torch.Tensor,
                       x0_hist: Optional[torch.Tensor], coef: torch.Tensor, step_idx: Optional[torch.Tensor]):
    n, _, f, h, w = x.shape
    _lib.call("aab_cfg_scheduler_step", _ptr(eps), ldc, int(cfg), float(guidance), _ptr(x), _ptr(x_out), _ptr(x0_hist),
              _ptr(coef), _ptr(step_idx), n, f, h, w, _is_bf16(x), _stream())
    return x_out


def image_to_nhwc8(img: torch.Tensor) -> torch.Tensor:
    n, c, h, w = img.shape
    out = torch.empty((n, h, w, 8), device=img.device, dtype=img.dtype)
    _lib.call("aab_image_to_nhwc8", _ptr(img), img.stride(0), img.stride(1), img.stride(2), img.stride(3), _ptr(out), n, c,
              h, w, _is_bf16(img), _stream())
    return out


def image_to_nhwc16(img: torch.Tensor) -> torch.Tensor:
    """[N, C<=16, H, W] (any strides) -> channels-last [N, H, W, 16], zero padded."""
    n, c, h, w = img.shape
    out = torch.empty((n, h, w, 16), device=img.device, dtype=img.dtype)
    _lib.call("aab_image_to_nhwc16", _ptr(img), img.stride(0), img.stride(1), img.stride(2), img.stride(3), _ptr(out), n, c,
              h, w, _is_bf16(img), _stream())
    return out


def add_rowvec(x: torch.Tensor, vec: torch.Tensor, rows_per_vec: int, mod: int, mode: int = 0, mod2: int = 1,
               inplace: bool = False) -> torch.Tensor:
    """x[r] + vec[idx(r)] (fp32 vec rows).  mode 0: idx = (r // rows_per_vec) % mod; mode 1 (rows (b, f, s),
    S = rows_per_vec, F = mod2): idx = (b * S + s) % mod."""
    assert vec.dtype == torch.float32 and vec.stride(-1) == 1
    out = x if inplace else torch.empty((x.shape[0], x.shape[1]), device=x.device, dtype=x.dtype)
    _lib.call("aab_add_rowvec", _ptr(x), x.stride(0), _ptr(out), out.stride(0), _ptr(vec), vec.stride(0), x.shape[0],
              x.shape[1], rows_per_vec, mod, mode, mod2, _is_bf16(x), _stream())
    return out


def axpby(x: torch.Tensor, y: torch.Tensor, a: float, b: float) -> torch.Tensor:
    assert x.is_contiguous() and y.is_contiguous() and x.shape == y.shape
    out = torch.empty_like(x)
    _lib.call("aab_axpby", _ptr(x), _ptr(y), _ptr(out), x.numel(), float(a), float(b), _is_bf16(x), _stream())
    return out


def svd_out_finalize(y: torch.Tensor, b: int, f: int, h: int, w: int, dtype) -> torch.Tensor:
    out = torch.empty((b, f, 4, h, w), device=y.device, dtype=dtype)
    _lib.call("aab_svd_out_finalize", _ptr(y), y.stride(0), _ptr(out), b * f, h, w, 1 if dtype == torch.bfloat16 else 0,
              _stream())
    return out


def svd_in_assemble(x: torch.Tensor, img_lat: torch.Tensor, mask: torch.Tensor, sigma: float, cfg: bool) -> torch.Tensor:
    """x [B, F, 4, h, w], img_lat [B, 4, h, w], mask [h, w] (same 16-bit dtype) -> UNet input [(2)B*F, h, w, 16]."""
    b, f, _, h, w = x.shape
    assert x.is_contiguous() and img_lat.is_contiguous() and mask.is_contiguous() and mask.numel() == h * w
    out = torch.empty(((2 if cfg else 1) * b * f, h, w, 16), device=x.device, dtype=x.dtype)
    _lib.call("aab_svd_in_assemble", _ptr(x), _ptr(img_lat), _ptr(mask), 1.0 / math.sqrt(sigma * sigma + 1.0), _ptr(out), b, f,
              h, w, int(cfg), _is_bf16(x), _stream())
    return out


def svd_in_assemble_frames(x: torch.Tensor, cond: torch.Tensor, mask: Optional[torch.Tensor], sigma: float, cfg: bool,
                           zero_uncond: bool) -> torch.Tensor:
    """General UNet input assembly of the SVD loops (TextStableVideoDiffusionPipeline): x [B, F, 4, h, w]; cond [Hc, B, F', 4, h, w]
    with Hc in (1, 2) CFG halves and F' in (1, F) frames (1 = broadcast); mask [B, F, h, w] or None (8-channel UNet).
    -> [(2)B*F, h, w, 16] channels-last (9 or 8 channels used)."""
    b, f, _, h, w = x.shape
    assert x.is_contiguous() and cond.is_contiguous() and cond.dim() == 6 and cond.shape[1] == b and cond.shape[3:] == (4, h, w)
    hc, _, fc = cond.shape[:3]
    assert hc in (1, 2) and fc in (1, f)
    if mask is not None:
        assert mask.is_contiguous() and tuple(mask.shape) == (b, f, h, w) and mask.dtype == x.dtype
    out = torch.empty(((2 if cfg else 1) * b * f, h, w, 16), device=x.device, dtype=x.dtype)
    _lib.call("aab_svd_in_assemble_frames", _ptr(x), _ptr(cond), cond.stride(0) if hc == 2 else 0, cond.stride(1),
              cond.stride(2) if fc == f and f > 1 else 0, int(zero_uncond), _ptr(mask), 0 if mask is None else mask.stride(0),
              0 if mask is None else mask.stride(1), 1.0 / math.sqrt(sigma * sigma + 1.0), _ptr(out), b, f, h, w, int(cfg),
              _is_bf16(x), _stream())
    return out


def svd_cfg_euler_step(pred: torch.Tensor, cfg: bool, gs: Optional[torch.Tensor], x: torch.Tensor, sigma: float,
                       sigma_next: float) -> torch.Tensor:
    b, f, _, h, w = x.shape
    out = torch.empty_like(x)
    _lib.call("aab_svd_cfg_euler_step", _ptr(pred), pred.stride(0), int(cfg), _ptr(gs), _ptr(x), _ptr(out), float(sigma),
              float(sigma_next), b, f, h, w, _is_bf16(x), _stream())
    return out


def vae_enc_finalize(mom: torch.Tensor, wq, bq, scale, b, f, h, w) -> torch.Tensor:
    """conv_out output [b*f*h*w, >=8] -> quant_conv -> moments [b, 8, f, h, w]."""
    out = torch.empty((b, 8, f, h, w), device=mom.device, dtype=mom.dtype)
    _lib.call("aab_vae_enc_finalize", _ptr(mom), mom.stride(0), _ptr(wq), _ptr(bq), float(scale), _ptr(out), b, f, h, w,
              _is_bf16(mom), _stream())
    return out


def add_noise(x0: torch.Tensor, noise: torch.Tensor, sa: float, sb: float) -> torch.Tensor:
    """x0 [b, c, 1|f, h, w], noise [b, c, f, h, w] (same 16-bit dtype, contiguous) -> sa * repeat(x0) + sb * noise."""
    b, c, f, h, w = noise.shape
    assert x0.dtype == noise.dtype and x0.shape[2] in (1, f) and x0.shape[:2] == noise.shape[:2]
    x0, noise = x0.contiguous(), noise.contiguous()
    out = torch.empty_like(noise)
    _lib.call("aab_add_noise", _ptr(x0), _ptr(noise), float(sa), float(sb), _ptr(out), b * c, f, x0.shape[2], h * w,
              _is_bf16(noise), _stream())
    return out


def vae_dec_in(lat: torch.Tensor, inv_scale, wp, bp) -> torch.Tensor:
    b, _, f, h, w = lat.shape
    out = torch.empty((b * f, h, w, 8), device=lat.device, dtype=lat.dtype)
    _lib.call("aab_vae_dec_in", _ptr(lat), float(inv_scale), _ptr(wp), _ptr(bp), _ptr(out), b, f, h, w, _is_bf16(lat),
              _stream())
    return out


def vae_dec_finalize(y: torch.Tensor, b, f, h, w, bf16: bool) -> torch.Tensor:
    out = torch.empty((b, 3, f, h, w), device=y.device, dtype=torch.float32)
    _lib.call("aab_vae_dec_finalize", _ptr(y), y.stride(0), _ptr(out), b, f, h, w, int(bf16), _stream())
    return out


def vae_dec_finalize_u8(y: torch.Tensor, b, f, h, w, bf16: bool, round_half_even: bool = False) -> torch.Tensor:
    """conv_out result -> uint8 frames [f, h, b*w, 3] (diffusers tensor2vid layout and rounding: the scaled value is
    truncated).  `round_half_even`: the SVD pipelines' `postprocess(..., "pil")` rounding instead, numpy's
    `((x / 2 + 0.5).clamp(0, 1) * 255).round()` on the fp32 product (bit 1 of the entry point's flag)."""
    out = torch.empty((f, h, b * w, 3), device=y.device, dtype=torch.uint8)
    _lib.call("aab_vae_dec_finalize_u8", _ptr(y), y.stride(0), _ptr(out), b, f, h, w,
              int(bf16) | (2 if round_half_even else 0), _stream())
    return out


# ---------------------------------------------------------------------------------------------- transparent-video branch
def video_f32_to_nhwc8(video: torch.Tensor, dtype) -> torch.Tensor:
    """fp32 video [b, c<=8, f, H, W] (any strides) -> channels-last 16-bit [b*f, H, W, 8], zero padded
    (models/pipeline_stage2.py:305)."""
    assert video.dtype == torch.float32 and video.dim() == 5
    b, c, f, h, w = video.shape
    out = torch.empty((b * f, h, w, 8), device=video.device, dtype=dtype)
    sb, sc, sf, sy, sx = video.stride()
    _lib.call("aab_video_f32_to_nhwc8", _ptr(video), sb, sc, sf, sy, sx, _ptr(out), b, c, f, h, w,
              1 if dtype == torch.bfloat16 else 0, _stream())
    return out


def rgba_finalize_u8(y: torch.Tensor, pixels: int, bf16: bool) -> torch.Tensor:
    """alpha decoder conv_out result [>= pixels, >= 4] fp32 -> uint8 [pixels, 4] (models/pipeline_stage2.py:311-324)."""
    assert y.dtype == torch.float32 and y.shape[0] >= pixels and y.shape[1] >= 4
    out = torch.empty((pixels, 4), device=y.device, dtype=torch.uint8)
    _lib.call("aab_rgba_finalize_u8", _ptr(y), y.stride(0), _ptr(out), pixels, int(bf16), _stream())
    return out


def pad_cols(x: torch.Tensor, dst_cols: int) -> torch.Tensor:
    """[rows, C] -> [rows, dst_cols] with zero columns appended."""
    out = torch.empty((x.shape[0], dst_cols), device=x.device, dtype=x.dtype)
    _lib.call("aab_pad_cols", _ptr(x), x.stride(0), _ptr(out), x.shape[0], x.shape[1], dst_cols, _stream())
    return out


def cat_cols(x: torch.Tensor, x2: torch.Tensor) -> torch.Tensor:
    """Materialised channel concat [rows, C1 + C2] (two strided copies): used where the virtual concat of the implicit GEMM
    cannot be (C1 not a multiple of the 64-channel K block)."""
    _is_bf16(x)                                                   # 16-bit only: the second copy is addressed in 2-byte elements
    assert x2.dtype == x.dtype and x2.shape[0] == x.shape[0]
    c1, c2 = x.shape[1], x2.shape[1]
    out = torch.empty((x.shape[0], c1 + c2), device=x.device, dtype=x.dtype)
    _lib.call("aab_copy2d", _ptr(x), x.stride(0), _ptr(out), out.stride(0), x.shape[0], c1, _stream())
    _lib.call("aab_copy2d", _ptr(x2), x2.stride(0), C.c_void_p(out.data_ptr() + 2 * c1), out.stride(0), x2.shape[0], c2,
              _stream())
    return out
