"""CPU: argument checks of the attention and normalisation entry points (fake buffers, only calls that return before any
launch), the table of which GPU test covers each C-ABI entry point of include/aab200.h, and the AlphaBlender coefficient
the SVD UNet hands to `aab_axpby`."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "aab200.h")


# ---------------------------------------------------------------------------------------------- argument checks
@pytest.fixture(scope="module")
def buffers():
    from animate_anything_b200 import _lib
    lib = _lib.load()
    buf = (C.c_float * 4096)()
    p = C.c_void_p((C.addressof(buf) + 15) // 16 * 16)
    return lib, buf, p


def test_flash_attn_d64_rejects_bad_arguments_without_a_gpu(buffers):
    lib, _, p = buffers
    mis = C.c_void_p(p.value + 2)

    def fa(q=p, kv=p, out=p, ldq=192, ldkv=192, ld_out=64, q_bs=None, kv_bs=None, q_cols=192, kv_cols=192, q_col0=0,
           k_col0=64, v_col0=128, out_col0=0, nb=2, nb_kv=2, div=1, heads=1, lq=4, lk=4, bf=0):
        return lib.aab_flash_attn_d64(q, ldq, lq * ldq if q_bs is None else q_bs, q_cols, q_col0, kv, ldkv,
                                      lk * ldkv if kv_bs is None else kv_bs, kv_cols, k_col0, v_col0, out, ld_out, lq * ld_out,
                                      out_col0, nb, nb_kv, div, heads, lq, lk, 0.125, bf, None)
    assert fa(q=None) == 1 and fa(kv=None) == 1 and fa(out=None) == 1
    assert fa(lq=0) == 1 and fa(lk=0) == 1 and fa(heads=0) == 1 and fa(nb=0) == 1 and fa(nb_kv=0) == 1 and fa(div=0) == 1
    assert fa(ldq=196) == 1 and fa(ldkv=196) == 1 and fa(ld_out=68) == 1 and fa(out_col0=4) == 1   # strides / offset % 8
    assert fa(bf=3, lq=4, lk=8) == 1 and fa(bf=2, lq=129, lk=129) == 1                 # causal: lq == lk <= 128 only
    # misaligned bases and batch strides (TMA needs 16-byte addresses)
    assert fa(q=mis) == 1 and fa(kv=mis) == 1 and fa(out=mis) == 1
    assert fa(q_bs=4 * 192 + 4) == 1 and fa(kv_bs=4 * 192 + 4) == 1
    # heads outside the described columns: TMA would read zero fill and return wrong attention
    assert fa(heads=2) == 1                                                          # V: 128 + 2 x 64 > 192 columns
    assert fa(q_col0=160) == 1 and fa(k_col0=136) == 1 and fa(v_col0=136) == 1
    assert fa(q_col0=-8) == 1 and fa(k_col0=-8) == 1 and fa(v_col0=-64) == 1
    assert fa(q_cols=56) == 1 and fa(kv_cols=184) == 1
    # a query batch whose K/V batch b / kv_batch_div does not exist
    assert fa(nb=3, nb_kv=2) == 1 and fa(nb=5, nb_kv=2, div=2) == 1 and fa(nb=7, nb_kv=2, div=3) == 1


def test_temporal_attn_d64_rejects_bad_arguments_without_a_gpu(buffers):
    lib, _, p = buffers
    mis = C.c_void_p(p.value + 8)

    def ta(qkv=p, out=p, ld=384, ld_out=128, q_col0=0, k_col0=128, v_col0=256, b=1, t=4, hw=2, heads=2):
        return lib.aab_temporal_attn_d64(qkv, ld, q_col0, k_col0, v_col0, out, ld_out, b, t, hw, heads, 0.125, 0, None)
    assert ta(qkv=None) == 1 and ta(out=None) == 1
    assert ta(t=0) == 1 and ta(t=33) == 1
    assert ta(b=0) == 1 and ta(hw=0) == 1 and ta(heads=0) == 1 and ta(b=-1) == 1
    assert ta(ld=388) == 1 and ta(ld_out=132) == 1 and ta(k_col0=132) == 1
    assert ta(qkv=mis) == 1 and ta(out=mis) == 1
    assert ta(v_col0=320) == 1 and ta(q_col0=264) == 1 and ta(heads=3) == 1          # a head past the end of a qkv row
    assert ta(ld_out=64) == 1                                                          # output row narrower than heads x 64
    assert ta(q_col0=-8) == 1


def test_groupnorm_rejects_bad_arguments_without_a_gpu(buffers):
    """Both GroupNorm entry points move the activations in 16-byte pieces: a base that is not 16-byte aligned (a column view
    at an odd offset) returns 1 instead of faulting; so do missing affine parameters and empty extents."""
    lib, _, p = buffers
    mis = C.c_void_p(p.value + 2)

    def gn(x1=p, x2=None, y=p, gamma=p, beta=p, ws=p, c1=64, c2=0, ld1=64, ld2=64, ldy=64, samples=2, rows=256, groups=32):
        return lib.aab_groupnorm(x1, ld1, c1, x2, ld2, c2, samples, rows, groups, gamma, beta, 1e-5, 1, y, ldy, ws, 0, None)

    def gnc(x1=p, x2=None, y=p, gamma=p, beta=p, ws=p, st2=p, c1=64, c2=0, samples=2, rows=256, groups=32):
        return lib.aab_groupnorm_colstats(x1, 64, c1, p, x2, 64, c2, st2, samples, rows, groups, gamma, beta, 1e-5, 1, y, 64,
                                          ws, 0, None)
    for f in (gn, gnc):
        assert f(x1=mis) == 1 and f(y=mis) == 1 and f(x2=mis, c2=64) == 1 and f(x2=C.c_void_p(p.value + 8), c2=64) == 1
        assert f(gamma=None) == 1 and f(beta=None) == 1
        assert f(samples=0) == 1 and f(samples=-1) == 1 and f(rows=0) == 1 and f(samples=4097) == 1
        assert f(x1=None) == 1 and f(y=None) == 1 and f(ws=None) == 1 and f(x2=None, c2=64) == 1
        assert f(groups=0) == 1 and f(groups=3) == 1 and f(groups=512, c1=1024) == 1
    assert gn(ld1=68) == 1 and gn(ldy=68) == 1 and gn(c1=60) == 1 and gn(x2=p, c2=64, ld2=68) == 1
    assert gnc(rows=200) == 1 and gnc(x2=p, c2=64, st2=None) == 1                    # 128-row tiles; second statistics
    assert lib.aab_groupnorm_workspace_bytes(4097, 256, 64, 32) == -1
    assert lib.aab_groupnorm_workspace_bytes(4096, 256, 64, 32) > 0


def test_layernorm_rejects_bad_arguments_without_a_gpu(buffers):
    """x / y move as uint4 and gamma / beta as float4: each must be 16-byte aligned."""
    lib, _, p = buffers

    def ln(x=p, y=p, gamma=p, beta=p, ldx=64, ldy=64, rows=4, c=64):
        return lib.aab_layernorm(x, ldx, y, ldy, gamma, beta, rows, c, 1e-5, 0, None)
    for off in (2, 4, 8):
        mis = C.c_void_p(p.value + off)
        assert ln(x=mis) == 1 and ln(y=mis) == 1 and ln(gamma=mis) == 1 and ln(beta=mis) == 1, off
    assert ln(gamma=None) == 1 and ln(beta=None) == 1 and ln(x=None) == 1 and ln(y=None) == 1
    assert ln(rows=0) == 1 and ln(rows=-3) == 1
    assert ln(c=60) == 1 and ln(c=2056) == 1 and ln(ldx=68) == 1 and ln(ldy=68) == 1


def test_softmax_rows_rejects_bad_arguments_without_a_gpu(buffers):
    lib, _, p = buffers

    def sm(s=p, pr=p, lds=16, ldp=16, rows=4, l=10):
        return lib.aab_softmax_rows(s, lds, pr, ldp, rows, l, 0, None)
    assert sm(s=None) == 1 and sm(pr=None) == 1
    assert sm(rows=0) == 1 and sm(rows=-1) == 1 and sm(l=0) == 1 and sm(l=-5) == 1
    assert sm(lds=9) == 1 and sm(ldp=9) == 1                            # a score / probability row shorter than l


def test_igemm_rejects_undefined_flags_without_a_gpu(buffers):
    """A flags word with a bit outside the defined AAB_F_* set (32 and 16384 once selected thread-block clusters) returns 1
    before any CUDA call, instead of launching something other than what the caller asked for."""
    from animate_anything_b200 import _lib
    lib, _, p = buffers
    d = _lib.IgemmDesc()
    d.a = d.b = d.out = p.value
    d.kc, d.num_taps, d.n, d.block_n, d.out_scale = 64, 1, 64, 64, 1.0
    for i in range(4):
        d.dim_d[i], d.box[i] = (128, 128) if i == 0 else (1, 1)
    for bit in (32, 16384, 1 << 30):
        d.flags = bit
        assert lib.aab_igemm(C.byref(d), None) == 1, bit


# ---------------------------------------------------------------------------------------------- coverage table
# Every entry point of include/aab200.h -> (GPU test that checks it directly, note).  A test id is "file::function"; a row
# without one says why there is no direct test.  A new entry point without a row fails test_every_entry_point_has_a_row.
KC = "test_gpu_kernel_contracts.py"
AE = "test_gpu_attention_edges.py"
NC = "test_gpu_norm_contracts.py"
COVERAGE = {
    "aab_igemm": ("test_gpu_igemm.py::test_linear_plain", "plus conv / tconv / batched / 256-column variants in that file"),
    "aab_igemm_emits_colstats": ("test_gpu_norm_elem.py::test_igemm_epilogue_column_statistics", ""),
    "aab_flash_attn_d64": (f"{AE}::test_flash_d64_tail_lengths", "plus score patterns, leakage, causal, arguments"),
    "aab_flash_attn_d80": (f"{AE}::test_flash_d80_tail_lengths", "plus test_gpu_clip_vision.py::test_flash_d80_self"),
    "aab_clip_image_prep": ("test_gpu_clip_vision.py::test_clip_image_prep_matches_restatement", ""),
    "aab_temporal_attn_d64": (f"{AE}::test_temporal_frame_counts", "plus persistent loop, large logits"),
    "aab_groupnorm_workspace_bytes": (f"{NC}::test_groupnorm_workspace_sample_counts",
                                      "host-side size query, used by every GroupNorm; plus test_groupnorm_chunk_cap"),
    "aab_groupnorm": (f"{NC}::test_groupnorm_call_sites",
                      "plus chunk cap, concat split inside a group, strided input, workspace, large mean"),
    "aab_groupnorm_colstats": (f"{NC}::test_groupnorm_column_statistics", "plus concat split inside a group, large mean"),
    "aab_layernorm": (f"{NC}::test_layernorm_instances", "plus constant rows, token-0 rows"),
    "aab_softmax_rows": (f"{NC}::test_softmax_rows_padding_and_patterns", "plus test_vae_mid_attention_chain"),
    "aab_unet_in_assemble": (f"{KC}::test_unet_in_assemble_per_sample_masks",
                             "plus test_gpu_norm_elem.py::test_unet_boundary_kernels"),
    "aab_unet_out_finalize": ("test_gpu_norm_elem.py::test_unet_boundary_kernels", ""),
    "aab_timestep_embed": (f"{KC}::test_timestep_embed", ""),
    "aab_embed_tokens": (f"{KC}::test_embed_tokens", ""),
    "aab_image_to_nhwc16": (f"{KC}::test_image_to_nhwc16", ""),
    "aab_add_rowvec": (f"{KC}::test_add_rowvec", ""),
    "aab_axpby": (f"{KC}::test_axpby", ""),
    "aab_svd_out_finalize": (f"{KC}::test_svd_out_finalize", ""),
    "aab_svd_in_assemble": (f"{KC}::test_svd_in_assemble", ""),
    "aab_svd_in_assemble_frames": ("test_gpu_svd.py::test_svd_in_assemble_frames_kernel", ""),
    "aab_svd_cfg_euler_step": (f"{KC}::test_svd_cfg_euler_step", ""),
    "aab_geglu": ("test_gpu_norm_elem.py::test_unet_boundary_kernels", ""),
    "aab_upsample2x": ("test_gpu_norm_elem.py::test_unet_boundary_kernels", ""),
    "aab_upsample_nearest": (f"{KC}::test_upsample_nearest_unet_sizes", "plus test_upsample_nearest_sweep"),
    "aab_pad_br": (f"{KC}::test_pad_to_even", ""),
    "aab_copy2d": (f"{KC}::test_copy2d_both_paths", ""),
    "aab_dup_rows": (f"{KC}::test_dup_rows", ""),
    "aab_transpose": ("test_gpu_norm_elem.py::test_softmax_rows_and_transpose", f"plus {NC}::test_vae_mid_attention_chain"),
    "aab_cfg_scheduler_step": (f"{KC}::test_cfg_scheduler_step_coefficients",
                               "plus test_gpu_norm_elem.py::test_cfg_scheduler_step"),
    "aab_image_to_nhwc8": ("test_gpu_norm_elem.py::test_vae_boundary_kernels", ""),
    "aab_vae_enc_finalize": (f"{KC}::test_vae_enc_finalize_scaled",
                             "scale = 1: test_gpu_norm_elem.py::test_vae_boundary_kernels"),
    "aab_vae_dec_in": (f"{KC}::test_vae_dec_in", ""),
    "aab_vae_dec_finalize": (f"{KC}::test_vae_dec_finalize_every_value", ""),
    "aab_vae_dec_finalize_u8": (f"{KC}::test_vae_dec_finalize_u8_every_value", "both roundings, every finite 16-bit value"),
    "aab_add_noise": ("test_gpu_pipeline.py::test_common_ddpm_forward_timesteps_bit_exact", ""),
    "aab_video_f32_to_nhwc8": ("test_gpu_transparent.py::test_video_f32_to_nhwc8_and_rgba_finalize_bit_exact", ""),
    "aab_rgba_finalize_u8": ("test_gpu_transparent.py::test_video_f32_to_nhwc8_and_rgba_finalize_bit_exact", ""),
    "aab_pad_cols": ("test_gpu_transparent.py::test_pad_cols_and_cat_cols", ""),
    "aab_cast_f32": (f"{KC}::test_cast_f32_special_values", "no caller in the package; tested so that it can be used"),
    "aab_num_sms": (None, "host query of the device's SM count, no kernel: nothing to compare"),
}


def _header_entry_points():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.findall(r"^\s*(?:int|long)\s+(aab_\w+)\s*\(", text, flags=re.M)


def test_every_entry_point_has_a_row():
    names = _header_entry_points()
    assert len(names) == len(set(names)) and len(names) >= 40, names
    missing = sorted(set(names) - set(COVERAGE))
    stale = sorted(set(COVERAGE) - set(names))
    assert not missing, f"entry points without a row in COVERAGE: {missing}"
    assert not stale, f"rows for entry points the header no longer declares: {stale}"


@pytest.mark.parametrize("name", sorted(COVERAGE))
def test_coverage_row_names_a_gpu_test_or_a_reason(name):
    test_id, note = COVERAGE[name]
    if test_id is None:
        assert note, f"{name}: no test and no reason"
        return
    fname, func = test_id.split("::")
    src = open(os.path.join(ROOT, "tests", fname)).read()
    m = re.search(rf"^def {func}\(", src, flags=re.M)
    assert m, f"{name}: {test_id} does not exist"
    # the test (or its module) runs under -m gpu
    head = src[:m.start()].rsplit("\ndef ", 1)[-1]
    assert "pytestmark = pytest.mark.gpu" in src or "@pytest.mark.gpu" in head, f"{test_id} is not a GPU test"


# ---------------------------------------------------------------------------------------------- AlphaBlender coefficient
@pytest.mark.parametrize("mix", [0.5, -0.37, 1.3])
@pytest.mark.parametrize("switch", [False, True])
def test_alpha_blender_coefficient_is_fp32_sigmoid(mix, switch):
    """The SVD UNet passes alpha = sigmoid(mix_factor) in fp32 (not rounded to the model dtype) to `aab_axpby`; the other
    coefficient is 1 - alpha.  tests/test_gpu_kernel_contracts.py::test_axpby pins the kernel's roundings for such
    coefficients."""
    from animate_anything_b200.unet_spatio_temporal_condition import AlphaBlender, _alpha
    m = AlphaBlender(mix, "learned_with_images", switch_spatial_to_temporal_mix=switch)
    s = float(torch.sigmoid(torch.tensor(mix, dtype=torch.float32)).item())
    assert _alpha(m) == (1.0 - s if switch else s)
    for dt in (torch.float16, torch.bfloat16):
        assert s != float(torch.tensor(s).to(dt))                  # the 16-bit-rounded alpha would be a different value
