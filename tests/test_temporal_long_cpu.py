"""CPU: clips longer than 32 frames.  Argument checks of the long-clip temporal attention (bit 1 of is_bf16; fake buffers,
every call returns before a launch), the frame count -> kernel choice, and the host wiring of both UNets at 40 frames over
the plain-torch kernel stand-ins of tests/ops_emulation.py, with the long-clip wrapper emulated here."""
import ctypes as C
import math
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

from ops_emulation import emulated_ops  # noqa: E402
from oracle.composition import fill_deterministic  # noqa: E402


# ---------------------------------------------------------------------------------------------- argument checks
def test_long_clip_flag_rejects_bad_arguments_without_a_gpu():
    from animate_anything_b200 import _lib
    lib = _lib.load()
    buf = (C.c_float * 4096)()
    p = C.c_void_p((C.addressof(buf) + 15) // 16 * 16)
    mis = C.c_void_p(p.value + 8)

    def ta(qkv=p, out=p, ld=384, ld_out=128, q_col0=0, k_col0=128, v_col0=256, b=1, t=40, hw=2, heads=2, flags=2):
        return lib.aab_temporal_attn_d64(qkv, ld, q_col0, k_col0, v_col0, out, ld_out, b, t, hw, heads, 0.125, flags, None)
    for bf in (0, 1):
        f = 2 | bf
        assert ta(t=129, flags=f) == 1 and ta(t=0, flags=f) == 1 and ta(t=-1, flags=f) == 1
        assert ta(t=33, flags=bf) == 1 and ta(t=128, flags=bf) == 1                     # without bit 1: 32 frames at most
        assert ta(qkv=None, flags=f) == 1 and ta(out=None, flags=f) == 1
        assert ta(b=0, flags=f) == 1 and ta(hw=0, flags=f) == 1 and ta(heads=0, flags=f) == 1
        assert ta(ld=388, flags=f) == 1 and ta(ld_out=132, flags=f) == 1 and ta(k_col0=132, flags=f) == 1
        assert ta(qkv=mis, flags=f) == 1 and ta(out=mis, flags=f) == 1
        assert ta(v_col0=320, flags=f) == 1 and ta(heads=3, flags=f) == 1 and ta(ld_out=64, flags=f) == 1
        assert ta(q_col0=-8, flags=f) == 1
    for flags in (4, 5, 6, 7, 8, 11, 16, -1, -2, 1 << 30):                              # unknown bits
        assert ta(flags=flags) == 1 and ta(t=4, flags=flags) == 1, flags


# ---------------------------------------------------------------------------------------------- kernel choice
def test_frame_count_picks_the_kernel(monkeypatch):
    from animate_anything_b200 import ops
    calls = []
    monkeypatch.setattr(ops, "temporal_attn_d64", lambda *a: calls.append(("d64", a[2])))
    monkeypatch.setattr(ops, "temporal_attn_long", lambda *a: calls.append(("long", a[2])))
    for t in (1, 32, 33, 128):
        ops.temporal_attn(None, 1, t, 4, 1, 0, 64, 128)
    assert calls == [("d64", 1), ("d64", 32), ("long", 33), ("long", 128)]
    with pytest.raises(NotImplementedError, match="128 frames"):
        ops.temporal_attn(None, 1, 129, 4, 1, 0, 64, 128)
    assert len(calls) == 4 and ops.TEMPORAL_MAX_FRAMES == 128


def test_both_unets_reject_129_frames_before_any_work():
    """Both forwards raise before their weights are prepared or a kernel is called (no GPU needed to see it)."""
    from animate_anything_b200.unet_3d_condition_mask import UNet3DConditionModel
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    m = UNet3DConditionModel(**UNET_CFG).eval()
    with pytest.raises(NotImplementedError, match="128 frames"):
        m(torch.zeros(1, 4, 128, 16, 16), 1, torch.zeros(1, 77, 128), condition_latent=torch.zeros(1, 4, 1, 16, 16),
          mask=None)
    assert m.__dict__.get("_aab_prepared") is None
    s = UNetSpatioTemporalConditionModel(**SVD_CFG).eval()
    with pytest.raises(NotImplementedError, match="128 frames"):
        s(torch.zeros(2, 129, 9, 8, 16), 1.0, torch.zeros(2, 1, 96), torch.zeros(2, 3))
    assert s.__dict__.get("_aab_prepared") is None


# ---------------------------------------------------------------------------------------------- host wiring at 40 frames
UNET_CFG = dict(sample_size=16, block_out_channels=(64, 128, 256, 256), attention_head_dim=64, cross_attention_dim=128,
                motion_mask=True, motion_strength=True)
SVD_CFG = dict(in_channels=9, block_out_channels=(64, 128, 128, 128), num_attention_heads=(1, 2, 2, 2), cross_attention_dim=96,
               addition_time_embed_dim=32, projection_class_embeddings_input_dim=96, num_frames=4, sample_size=16)


def _attn_long(calls):
    """Stand-in for ops.temporal_attn_long: float64 softmax attention over t for every (b, pixel, head)."""
    def run(qkv, b, t, hw, heads, q_col0, k_col0, v_col0):
        assert 33 <= t <= 128
        calls.append(t)

        def pick(col0):
            return qkv[:, col0:col0 + heads * 64].double().view(b, t, hw, heads, 64).permute(0, 2, 3, 1, 4)
        q, k, v = pick(q_col0), pick(k_col0), pick(v_col0)
        p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(64.0), dim=-1)
        return (p @ v).permute(0, 3, 1, 2, 4).reshape(b * t * hw, heads * 64).float()
    return run


def _host_prepared(m):
    m.__dict__["_aab_prepared"] = m._build_prepared(torch.float32, torch.device("cpu"))


def test_unet3d_host_wiring_40_frames(monkeypatch):
    from oracle.composition import OracleUNet3D
    from animate_anything_b200 import ops
    from animate_anything_b200.unet_3d_condition_mask import UNet3DConditionModel
    from make_golden import fp16_inputs
    m = fill_deterministic(UNet3DConditionModel(**UNET_CFG).eval(), seed=0)
    m.load_state_dict({k: v.half().float() for k, v in m.state_dict().items()})
    o = OracleUNet3D(**{k: v for k, v in UNET_CFG.items() if k != "sample_size"}).eval()
    o.load_state_dict(m.state_dict())
    inp = fp16_inputs(b=1, f=40, hw=8, lk=7, cdim=128)
    calls = []
    with emulated_ops():
        monkeypatch.setattr(ops, "temporal_attn_long", _attn_long(calls))
        _host_prepared(m)
        out = m(inp["sample"], 37, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"],
                motion=torch.tensor([4.0])).sample
    with torch.no_grad():
        ref = o(inp["sample"], 37, inp["ehs"], inp["cond"], inp["mask"], motion=torch.tensor([4.0]))
    assert calls and set(calls) == {41}
    assert out.shape == ref.shape == (1, 4, 40, 8, 8)
    err = float((out - ref).abs().max())
    assert err < 5e-4 * max(1.0, float(ref.abs().mean())), err


def test_svd_unet_host_wiring_40_frames(monkeypatch):
    from oracle.composition import UNetSpatioTemporalConditionModel as OUNet
    from animate_anything_b200 import ops
    from animate_anything_b200.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel
    o = fill_deterministic(OUNet(**SVD_CFG).eval(), seed=0)
    m = UNetSpatioTemporalConditionModel(**SVD_CFG).eval()
    m.load_state_dict(o.state_dict(), strict=True)
    g = torch.Generator().manual_seed(3)
    b, nf, h, w = 2, 40, 8, 8
    x = torch.randn(b, nf, 9, h, w, generator=g)
    emb = torch.randn(1, 1, 96, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    ids = torch.tensor([[6.0, 127.0, 0.02]] * 2)
    t = torch.tensor(1.6378)
    with torch.no_grad():
        ref = o(x, t, ehs, ids, return_dict=False)[0]
    calls = []
    with emulated_ops():
        monkeypatch.setattr(ops, "temporal_attn_long", _attn_long(calls))
        _host_prepared(m)
        out = m(x, t, ehs, ids).sample
    assert calls and set(calls) == {40}
    assert out.shape == ref.shape == (b, nf, 4, h, w)
    err = float((out - ref).abs().max())
    assert err < 5e-4 * max(1.0, float(ref.abs().mean())), err
