"""Which implicit-GEMM launches of a config-2 UNet forward take two CTAs per SM (`ops.pick_two_cta`), without a GPU."""
from animate_anything_b200 import ops


def test_two_cta_rule_on_config2_shapes():
    pick = ops.pick_two_cta
    # 1-tap transformer linears at 64x64 (1088 m-tiles, K = 320) and 32x32 (272 m-tiles, K = 640): 64-column tiles
    assert pick(320, 1088, 320, 1) == 64 and pick(960, 1088, 320, 1) == 64
    assert pick(640, 272, 640, 1) == 64 and pick(1920, 272, 640, 1) == 64
    # GEGLU (needs 128-column tiles), K > 640, 3x3 / temporal taps, fewer m-tiles than two CTAs on every SM, N < 320
    assert pick(1280, 1088, 320, 1, geglu=True) == 0
    assert pick(320, 1088, 1280, 1) == 0 and pick(1280, 68, 1280, 1) == 0
    assert pick(320, 1088, 960, 3) == 0 and pick(320, 1088, 2880, 9) == 0
    assert pick(320, 263, 320, 1) == 0 and pick(320, 264, 320, 1) == 64
    assert pick(64, 8192, 64, 1) == 0 and pick(1280, 2, 320, 1) == 0
