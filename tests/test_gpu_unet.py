"""GPU parity of the sm_90a UNet3DConditionModel.forward against the oracle (fp32, same 16-bit-rounded weights/inputs).

Three error levels are reported separately (SURVEY.md section 7 'fp16 tolerance'): per kernel (test_gpu_igemm/attention/
norm_elem: rtol=1e-3 fp16), single forward (here), full loop (test_gpu_pipeline).  For a whole forward the yard-stick is
the stock PyTorch fp16 execution of the same op sequence (oracle.half() on cuDNN/cuBLAS): our error vs the fp32 oracle
must not exceed 1.5x that of the stock fp16 stack (+ a small floor)."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from util import report  # noqa: E402

pytestmark = pytest.mark.gpu


def _models(cfg, dtype):
    from oracle.composition import OracleUNet3D, fill_deterministic
    from animate_anything_b200.unet_3d_condition_mask import UNet3DConditionModel
    ocfg = {k: v for k, v in cfg.items() if k != "sample_size"}
    oracle = fill_deterministic(OracleUNet3D(**ocfg).eval(), seed=0)
    sd16 = {k: v.to(dtype) for k, v in oracle.state_dict().items()}
    oracle.load_state_dict({k: v.float() for k, v in sd16.items()})      # fp32 math on 16-bit-rounded weights
    ours = UNet3DConditionModel(**cfg).eval()
    missing, unexpected = ours.load_state_dict(sd16, strict=True)
    return oracle.cuda(), ours.to(dtype).cuda()


def _inputs(b, f, hw, lk, cdim, dtype, seed=1):
    g = torch.Generator().manual_seed(seed)
    d = dict(sample=torch.randn(b, 4, f, hw, hw, generator=g), cond=torch.randn(b, 4, 1, hw, hw, generator=g),
             ehs=torch.randn(b, lk, cdim, generator=g), mask=(torch.rand(1, 1, 1, hw, hw, generator=g) > 0.5).float())
    return {k: v.to(dtype).cuda() for k, v in d.items()}


def _to_nchw(x, g):
    return x.float().reshape(g.n, g.h, g.w, -1).permute(0, 3, 1, 2)


def _run_case(cfg, dtype, b, f, hw, lk, timestep=500, motion=4.0, trace=True):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _models(cfg, dtype)
    inp = _inputs(b, f, hw, lk, cfg.get("cross_attention_dim", 1024), dtype)
    mot = torch.tensor([motion], device="cuda")
    captured = {}
    hooks = []
    if trace:
        def mk(name):
            def hook(mod, args, out):
                o = out[0] if isinstance(out, tuple) else out
                captured[name] = (o.sample if hasattr(o, "sample") else o).detach().float()
            return hook
        for name in (["conv_in2", "transformer_in", "mid_block"] + [f"down_blocks.{i}" for i in range(4)] +
                     [f"up_blocks.{i}" for i in range(4)]):
            hooks.append(oracle.get_submodule(name).register_forward_hook(mk(name)))
    with torch.no_grad():
        ref = oracle(inp["sample"].float(), timestep, inp["ehs"].float(), inp["cond"].float(), inp["mask"].float(),
                     motion=mot)
    for h in hooks:
        h.remove()
    ours._trace = [] if trace else None
    ours.__dict__["_trace"] = ours._trace
    out = ours(inp["sample"], timestep, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot).sample
    torch.cuda.synchronize()
    if trace:
        for name, x, g in ours.__dict__["_trace"]:
            key = "conv_in2" if name == "conv_in" else name
            if key in captured:
                report(f"  stage {name}", _to_nchw(x, g), captured[key], 1e-2, 1e-2)
    # stock fp16/bf16 torch execution of the same op sequence = the yard-stick
    with torch.no_grad():
        stock = oracle.to(dtype)(inp["sample"], timestep, inp["ehs"], inp["cond"], inp["mask"], motion=mot).float()
    e_ours = (out.float() - ref).abs()
    e_stock = (stock - ref).abs()
    scale = ref.abs().mean().item()
    print(f"forward {dtype}: ref|mean|={scale:.4f}  ours: max={e_ours.max().item():.4e} mean={e_ours.mean().item():.4e}"
          f"  stock-torch: max={e_stock.max().item():.4e} mean={e_stock.mean().item():.4e}")
    assert torch.isfinite(out).all()
    assert e_ours.mean().item() <= 1.5 * e_stock.mean().item() + 2e-4 * scale
    assert e_ours.max().item() <= 2.0 * e_stock.max().item() + 2e-3 * scale
    return e_ours, e_stock


SMALL = dict(sample_size=16, block_out_channels=(64, 128, 256, 256), attention_head_dim=64, cross_attention_dim=128,
             motion_mask=True, motion_strength=True)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_unet_small(dtype):
    _run_case(SMALL, dtype, b=2, f=4, hw=16, lk=77)


def test_unet_small_no_mask_single_frame_paths():
    """conv_in (4-ch) branch and motion=None branch (reference :414-419,:429-431)."""
    from oracle.composition import OracleUNet3D
    dtype = torch.float16
    cfg = dict(SMALL, motion_mask=False, motion_strength=False)
    _run_case(cfg, dtype, b=1, f=3, hw=16, lk=10, trace=False)


def test_unet_config1_fullsize():
    """BASELINE config 1 shapes on the full-size architecture: sample [1,4,8,32,32], text [1,77,1024], t=500, motion 4."""
    cfg = dict(sample_size=32, motion_mask=True, motion_strength=True)
    _run_case(cfg, torch.float16, b=1, f=8, hw=32, lk=77, trace=True)


def test_cfg_shared_prefix_matches_duplicated_batch():
    """The shared-prefix evaluation (one copy of the latents per CFG pair, duplicated at the first text cross-attention)
    equals the reference's `torch.cat([latents] * 2)` evaluation BIT FOR BIT: every kernel is batch-invariant (GEMM
    K-order, attention and norms are per row / per sample; the GroupNorm row partition depends on (rows, C) only)."""
    from util import check
    dtype = torch.float16
    oracle, ours = _models(SMALL, dtype)
    inp = _inputs(1, 4, 16, 77, SMALL["cross_attention_dim"], dtype)
    g = torch.Generator().manual_seed(9)
    ehs = torch.randn(2, 77, SMALL["cross_attention_dim"], generator=g).to(dtype).cuda()
    mot = torch.tensor([4.0], device="cuda")
    dup = ours(inp["sample"].expand(2, -1, -1, -1, -1), 321, ehs, condition_latent=inp["cond"].expand(2, -1, -1, -1, -1),
               mask=inp["mask"], motion=mot).sample
    shared = ours(inp["sample"], 321, ehs, condition_latent=inp["cond"], mask=inp["mask"], motion=mot,
                  _cfg_shared_prefix=True).sample
    assert shared.shape == dup.shape == (2, 4, 4, 16, 16)
    assert torch.equal(shared, dup), f"shared prefix != duplicated batch, max diff {(shared.float() - dup.float()).abs().max()}"
    with torch.no_grad():
        ref = oracle(inp["sample"].float().expand(2, -1, -1, -1, -1), 321, ehs.float(),
                     inp["cond"].float().expand(2, -1, -1, -1, -1), inp["mask"].float(), motion=mot)
    check("cfg shared prefix vs fp32 oracle", shared, ref, 2e-2, 1e-2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_batch_invariance(dtype):
    """Sample i of a batched forward equals the forward of sample i alone, bit for bit (what makes the CFG halves
    split over two GPUs, parallel.py / pipeline.cfg_group, reproduce the single-GPU latents exactly)."""
    _, ours = _models(SMALL, dtype)
    inp = _inputs(2, 4, 16, 77, SMALL["cross_attention_dim"], dtype)
    mot = torch.tensor([4.0], device="cuda")
    both = ours(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot).sample
    for i in range(2):
        one = ours(inp["sample"][i:i + 1], 500, inp["ehs"][i:i + 1], condition_latent=inp["cond"][i:i + 1],
                   mask=inp["mask"], motion=mot).sample
        assert torch.equal(one[0], both[i]), f"sample {i}: max diff {(one[0].float() - both[i].float()).abs().max()}"


@pytest.mark.parametrize("name", ["unet_small_ref.pt", "unet_config1_ref.pt"])
def test_unet_matches_reference_golden(name):
    """The CUDA path against the committed output of the VERBATIM reference files (tests/golden/make_golden.py::
    product_shape_goldens: fp32 on CPU, fp16-rounded weights and inputs): SMALL config and BASELINE config 1 at full
    size.  Same yard-stick as _run_case (stock 16-bit torch execution of the op sequence)."""
    gold = torch.load(os.path.join(HERE, "golden", name), map_location="cpu")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dtype = torch.float16
    sh = gold["shape"]
    oracle, ours = _models(dict(gold["config"]), dtype)
    inp = _inputs(sh["b"], sh["f"], sh["hw"], sh["lk"], sh["cdim"], dtype)
    mot = torch.tensor([gold["motion"]], device="cuda")
    ref = gold["out"].cuda()
    scale = ref.abs().mean().item()
    out = ours(inp["sample"], gold["timestep"], inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot).sample
    with torch.no_grad():
        o32 = oracle(inp["sample"].float(), gold["timestep"], inp["ehs"].float(), inp["cond"].float(), inp["mask"].float(),
                     motion=mot)
        stock = oracle.to(dtype)(inp["sample"], gold["timestep"], inp["ehs"], inp["cond"], inp["mask"], motion=mot).float()
    e_or = (o32 - ref).abs().max().item()
    e_ours = (out.float() - ref).abs()
    e_stock = (stock - ref).abs()
    print(f"{name}: golden|mean|={scale:.4f} fp32 oracle on GPU vs golden max={e_or:.3e} | ours max={e_ours.max().item():.4e} "
          f"mean={e_ours.mean().item():.4e} | stock fp16 max={e_stock.max().item():.4e} mean={e_stock.mean().item():.4e}")
    # cuDNN / cuBLAS fp32 (TF32 off) vs the CPU kernels: accumulation-order noise only
    assert e_or <= 5e-3 * scale, "the fp32 oracle on the GPU must reproduce the CPU output of the reference files"
    assert torch.isfinite(out).all()
    assert e_ours.mean().item() <= 1.5 * e_stock.mean().item() + 2e-4 * scale
    assert e_ours.max().item() <= 2.0 * e_stock.max().item() + 2e-3 * scale


def test_prepare_to_host_conversion_matches_lazy():
    """`ModelBase.prepare_to` (weights converted to kernel layouts on the host, uploaded by memcpy) gives the same bits
    as the lazy on-device conversion."""
    from oracle.composition import OracleUNet3D, fill_deterministic
    from animate_anything_b200.unet_3d_condition_mask import UNet3DConditionModel
    dtype = torch.float16
    sd = {k: v.to(dtype) for k, v in fill_deterministic(OracleUNet3D(**{k: v for k, v in SMALL.items()
                                                                       if k != "sample_size"}).eval(), 0).state_dict().items()}
    a = UNet3DConditionModel(**SMALL).eval()
    a.load_state_dict(sd)
    a = a.to(dtype).cuda()
    b = UNet3DConditionModel(**SMALL).eval()
    b.load_state_dict(sd)
    b = b.to(dtype).prepare_to("cuda")
    assert b.__dict__["_aab_prepared"] is not None and b.device.type == "cuda"
    inp = _inputs(2, 4, 16, 77, SMALL["cross_attention_dim"], dtype)
    mot = torch.tensor([4.0], device="cuda")
    ya = a(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot).sample
    yb = b(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot).sample
    assert torch.equal(ya, yb)
    with pytest.raises(ValueError):      # per-batch values: 1, B (reference broadcast rule) -- 3 values for batch 2 is an error
        a(inp["sample"], torch.tensor([1.0, 2.0, 3.0]), inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot)


def test_unet_odd_latent_size_upsample_size_path():
    """Latent 15 x 17 (not a multiple of 8): the reference's `forward_upsample_size` interpolation (:377-383,486-491) and
    odd stride-2 convolutions, against the verbatim-reference golden."""
    from util import assert_vs_stock, record_parity
    gold = torch.load(os.path.join(HERE, "golden", "unet_small_oddsize_ref.pt"), map_location="cpu")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dtype = torch.float16
    oracle, ours = _models(dict(gold["config"]), dtype)
    inp = {k: v.to(dtype).cuda() for k, v in gold["inputs"].items()}
    mot = torch.tensor([gold["motion"]], device="cuda")
    ref = gold["out"].cuda()
    out = ours(inp["sample"], gold["timestep"], inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot).sample
    with torch.no_grad():
        o32 = oracle(inp["sample"].float(), gold["timestep"], inp["ehs"].float(), inp["cond"].float(), inp["mask"].float(),
                     motion=mot)
        stock = oracle.to(dtype)(inp["sample"], gold["timestep"], inp["ehs"], inp["cond"], inp["mask"], motion=mot).float()
    assert (o32 - ref).abs().max().item() <= 5e-3 * ref.abs().mean().item()
    assert out.shape == ref.shape == (1, 4, 3, 15, 17)
    assert_vs_stock(record_parity("unet SMALL fp16 odd 15x17", "output (golden)", out, ref, stock))


def test_unet_forward_keyword_branches():
    """`attention_mask` / `class_labels` are accepted and ignored like the reference forward does (its blocks never read the
    mask: models/unet_3d_blocks.py:340,489,720; fixture unet_forward_branches_ref.pt records the verbatim behaviour), and
    `timestep_cond` (:418-419, no motion value) goes through time_embedding.cond_proj."""
    dtype = torch.float16
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    oracle, ours = _models(SMALL, dtype)
    inp = _inputs(2, 4, 16, 77, 128, dtype)
    mot = torch.tensor([4.0], device="cuda")
    base = ours(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot).sample
    same = ours(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot,
                attention_mask=torch.ones(2, 77, device="cuda"), class_labels=torch.tensor([1, 2], device="cuda"),
                timestep_cond=torch.randn(2, 64, device="cuda")).sample          # a motion value overrides timestep_cond
    assert torch.equal(base, same)
    g = torch.Generator().manual_seed(8)
    for rows in (2, 1):
        tc = torch.randn(rows, 64, generator=g).to(dtype).cuda()
        out = ours(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=None,
                   timestep_cond=tc).sample
        with torch.no_grad():
            ref = oracle.float()(inp["sample"].float(), 500, inp["ehs"].float(), inp["cond"].float(), inp["mask"].float(),
                                 motion=None, timestep_cond=tc.float())
            stock = oracle.to(dtype)(inp["sample"], 500, inp["ehs"], inp["cond"], inp["mask"], motion=None,
                                     timestep_cond=tc).float()
        e, es, sc = (out.float() - ref).abs(), (stock - ref).abs(), ref.abs().mean().item()
        assert (out.float() - base.float()).abs().mean().item() > 1e-3            # the branch is live
        assert e.mean().item() <= 1.5 * es.mean().item() + 2e-4 * sc and e.max().item() <= 2.0 * es.max().item() + 2e-3 * sc
    with pytest.raises(ValueError):
        ours(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=None,
             timestep_cond=torch.randn(3, 64, device="cuda"))
    with pytest.raises(NotImplementedError):
        ours(inp["sample"], 500, inp["ehs"], condition_latent=inp["cond"], mask=inp["mask"], motion=mot,
             mid_block_additional_residual=torch.zeros(1, device="cuda"))
