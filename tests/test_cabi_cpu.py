"""CPU: the C-ABI library builds, loads, and exports every symbol include/aab200.h declares (no compute calls);
host-side helpers (tile-box selection, block-N heuristic, config capture, state_dict key parity) behave."""
import ctypes
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _declared():
    src = open(os.path.join(ROOT, "include", "aab200.h")).read()
    return sorted(set(re.findall(r"\b(?:int|long)\s+(aab_[a-z0-9_]+)\s*\(", src)))


def test_header_compiles_as_c():
    import subprocess
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write('#include "aab200.h"\nint main(void){ AabIgemmDesc d; (void)d; return 0; }\n')
        subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-c", c, "-o", os.path.join(d, "t.o")],
                       check=True)


def test_igemm_desc_mirror_matches_the_c_struct():
    """`_lib.IgemmDesc` has the size and field offsets of `AabIgemmDesc` as the C compiler lays it out: a mismatch would
    have the library read the caller's descriptor at the wrong offsets."""
    import subprocess
    import tempfile
    from animate_anything_b200 import _lib
    names = [f[0] for f in _lib.IgemmDesc._fields_]
    prints = "".join(f'printf("%zu\\n", offsetof(AabIgemmDesc, {n}));' for n in names)
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "t.c"), os.path.join(d, "t")
        open(c, "w").write('#include <stddef.h>\n#include <stdio.h>\n#include "aab200.h"\n'
                           f'int main(void){{ printf("%zu\\n", sizeof(AabIgemmDesc)); {prints} return 0; }}\n')
        subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got[0] == ctypes.sizeof(_lib.IgemmDesc)
    assert dict(zip(names, got[1:])) == {n: getattr(_lib.IgemmDesc, n).offset for n in names}


def test_library_loads_and_exports_all_symbols():
    from animate_anything_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/aab200.h but not exported"
    for n in _lib.EXPORTS:
        assert n in names, f"{n} bound in _lib.py but not declared in include/aab200.h"
    assert ctypes.sizeof(_lib.IgemmDesc) > 0


def test_missing_library_fails_loudly(monkeypatch):
    from animate_anything_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libaab200.so")
    with pytest.raises(_lib.AabError):
        _lib.load()


def test_cpu_model_refuses_to_run():
    """No CPU / fp32 fallback: the product model raises instead of silently computing with torch."""
    from animate_anything_b200.unet_3d_condition_mask import UNet3DConditionModel
    m = UNet3DConditionModel(block_out_channels=(64, 64, 64, 64), cross_attention_dim=64)
    with pytest.raises((TypeError, RuntimeError)):
        m(torch.zeros(1, 4, 2, 8, 8), 1, torch.zeros(1, 7, 64), condition_latent=torch.zeros(1, 4, 1, 8, 8), mask=None)
    with pytest.raises(RuntimeError):
        m.down_blocks[0].resnets[0](torch.zeros(1))


def test_pick_box_and_block_n():
    from animate_anything_b200 import ops
    for dims in [(64, 64, 34, 1), (8, 8, 34, 1), (32, 32, 34, 1), (4096, 17, 2, 1), (64, 17, 2, 1), (2, 1, 1, 1),
                 (512, 512, 16, 1), (139264, 1, 1, 1)]:
        box = ops.pick_box(dims)
        p = 1
        for b in box:
            assert b >= 1 and (b & (b - 1)) == 0
            p *= b
        assert p == 128, (dims, box)
    assert ops.pick_box((32, 1, 32, 34), fixed_one=(1,))[1] == 1
    assert ops.pick_block_n(1280, 1088) == 256
    assert ops.pick_block_n(1280, 10, geglu=True) in (128, 256)
    assert ops.pick_block_n(320, 1088) == 256
    assert ops.pick_block_n(1280, 17) == 256          # widest tile even with fewer tiles than SMs (measured 1.7x)
    assert ops.pick_block_n(2560, 2) == 64            # GEMV-like: spread weight rows
    assert ops.pick_block_n(320, 1088, k_total=320) == 128
    # UNet384's 32 / 64-channel levels: N <= 64 takes 64-column tiles
    assert ops.pick_block_n(64, 8192, k_total=576) == 64 and ops.pick_block_n(128, 8192, k_total=1152) == 256


def test_new_entry_points_reject_bad_arguments_without_a_gpu():
    """Argument checks of the round-2c entry points run before any CUDA call: status 1 (bad argument) on a box with no GPU."""
    import ctypes as C
    from animate_anything_b200 import _lib
    lib = _lib.load()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    assert lib.aab_video_f32_to_nhwc8(None, 0, 0, 0, 0, 0, p, 1, 3, 1, 8, 8, 1, None) == 1
    assert lib.aab_video_f32_to_nhwc8(p, 0, 0, 0, 0, 0, p, 1, 9, 1, 8, 8, 1, None) == 1            # more than 8 channels
    assert lib.aab_rgba_finalize_u8(p, 3, p, 16, 1, None) == 1                                      # needs 4 channels per pixel
    assert lib.aab_rgba_finalize_u8(p, 4, None, 16, 1, None) == 1
    assert lib.aab_pad_cols(p, 32, p, 4, 32, 16, None) == 1                                         # destination narrower than source
    assert lib.aab_pad_cols(p, 30, p, 4, 32, 64, None) == 1                                         # row stride not a multiple of 8


def test_column_statistics_tile_order_predicate():
    """`ops.igemm(stats=True)` only asks for the epilogue's column sums when m-tile i of the kernel's tile order is exactly the
    output rows [128 i, 128 i + 128): the GroupNorm finalize kernel adds a sample's tiles by index."""
    from animate_anything_b200 import ops
    ok = ops._tiles_cover_rows_in_order
    for dim_d in [(64, 64, 34, 1), (32, 32, 34, 1), (16, 16, 34, 1), (8, 8, 34, 1), (4096, 17, 2, 1), (256, 17, 2, 1),
                  (139264, 1, 1, 1), (512, 512, 16, 1)]:
        assert ok(dim_d, ops.pick_box(dim_d)), dim_d
    assert ok((32, 1, 32, 34), ops.pick_box((32, 1, 32, 34), fixed_one=(1,)))       # stride-2 conv through space-to-depth
    assert not ok((15, 17, 34, 1), ops.pick_box((15, 17, 34, 1)))                   # odd latent size: partial boxes
    assert not ok((64, 17, 2, 1), ops.pick_box((64, 17, 2, 1)))                     # 8 x 8 level of the temporal conv: 17 % 2
    assert not ok((100, 1, 1, 1), (128, 1, 1, 1))
    # simulate the kernel's tile decode and check the claim itself on a few shapes
    import itertools
    for dim_d in [(16, 16, 3, 1), (8, 8, 4, 1), (256, 5, 2, 1), (15, 17, 2, 1), (64, 3, 2, 1)]:
        box = ops.pick_box(dim_d)
        tiles = [-(-d // b) for d, b in zip(dim_d, box)]
        in_order = True
        for mt in range(tiles[0] * tiles[1] * tiles[2] * tiles[3]):
            m, cb = mt, []
            for i in range(4):
                cb.append((m % tiles[i]) * box[i])
                m //= tiles[i]
            rows = []
            for r in range(128):
                g, rr, valid = [], r, True
                for i in range(4):
                    g.append(cb[i] + rr % box[i])
                    rr //= box[i]
                    valid = valid and g[i] < dim_d[i]
                if valid:
                    rows.append(((g[3] * dim_d[2] + g[2]) * dim_d[1] + g[1]) * dim_d[0] + g[0])
            in_order = in_order and rows == list(range(128 * mt, 128 * mt + 128))
        assert in_order == ok(dim_d, box), (dim_d, box)


def test_state_dict_keys_match_reference_naming():
    """Keys follow utils/convert_diffusers_to_original_ms_text_to_video.py:18-169 naming (and equal the oracle's, which is
    pinned to the verbatim reference model by tests/golden)."""
    from animate_anything_b200.autoencoder_kl import AutoencoderKL
    from animate_anything_b200.unet_3d_condition_mask import UNet3DConditionModel
    from oracle.composition import AutoencoderKL as OVAE, OracleUNet3D
    cfg = dict(block_out_channels=(64, 64, 128, 128), cross_attention_dim=64, motion_mask=True, motion_strength=True)
    a = set(UNet3DConditionModel(**cfg).state_dict().keys())
    b = set(OracleUNet3D(**cfg).state_dict().keys())
    assert a == b
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "unet_tiny_ref.pt"))
    strip = lambda ks: {re.sub(r"\d+", "N", k) for k in ks}
    assert strip(gold["keys"]) == strip(a)
    for k in ("conv_in2.weight", "time_embedding.cond_proj.weight", "transformer_in.proj_in.weight",
              "down_blocks.0.temp_convs.0.conv1.2.weight", "down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight",
              "up_blocks.1.upsamplers.0.conv.weight", "mid_block.temp_attentions.0.proj_out.bias", "conv_norm_out.weight"):
        assert k in a
    vcfg = dict(block_out_channels=(64, 64, 64, 64), layers_per_block=1)
    assert set(AutoencoderKL(**vcfg).state_dict().keys()) == set(OVAE(**vcfg).state_dict().keys())


def test_save_and_from_pretrained_roundtrip(tmp_path):
    from animate_anything_b200.unet_3d_condition_mask import UNet3DConditionModel
    cfg = dict(sample_size=8, block_out_channels=(64, 64, 64, 64), cross_attention_dim=64, motion_mask=True)
    m = UNet3DConditionModel(**cfg)
    m.save_pretrained(str(tmp_path / "unet"))
    m2 = UNet3DConditionModel.from_pretrained(str(tmp_path), subfolder="unet", motion_strength=True)
    assert m2.config.motion_mask is True and m2.config.motion_strength is True and m2.config.sample_size == 8
    for (k1, v1), (k2, v2) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k1 == k2 and torch.equal(v1, v2)


def test_built_library_contains_hopper_tensor_core_and_tma_sass():
    """The shipped `libaab200.so` is sm_90a code whose SASS holds the Hopper tensor-core and TMA instructions the design
    claims: HGMMA = wgmma.mma_async (fp16 / bf16, implicit GEMM and flash attention), UTMALDG = cp.async.bulk.tensor load,
    WARPGROUP = the wgmma fence / commit / wait.  HMMA (mma.sync) only serves the T <= 32 temporal attention."""
    import shutil
    import subprocess
    from animate_anything_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        import pytest
        pytest.skip("cuobjdump not available")
    arch = subprocess.run([tool, "-lelf", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    assert "sm_90a" in arch, arch[:400]
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    count = {m: sass.count(m) for m in ("HGMMA", "UTMALDG", "WARPGROUP", "HMMA")}
    assert count["HGMMA"] >= 40 and count["UTMALDG"] >= 30 and count["WARPGROUP"] >= 20, count
