"""CPU: the host logic of the CLIP image tower mirror (clip_vision.CLIPVisionModelWithProjection) against the real
`transformers.CLIPVisionModelWithProjection`, executed over plain-torch stand-ins of the kernels; the restatement of
diffusers' image preprocessing that the GPU tests use as the kernel's oracle, pinned to torchvision / torch / transformers;
and the argument checks of the two new C-ABI entry points (no GPU needed)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import clip_vision_emulation as cve  # noqa: E402

SMALL = dict(hidden_size=160, intermediate_size=640, projection_dim=96, num_hidden_layers=3, num_attention_heads=2,
             image_size=224, patch_size=14)


def hf_vision(seed=0, act="gelu", **over):
    """transformers CLIPVisionModelWithProjection with random weights scaled so that every layer matters."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    torch.manual_seed(seed)
    cfg = CLIPVisionConfig(**{**SMALL, **over}, hidden_act=act)
    m = CLIPVisionModelWithProjection(cfg).eval()
    with torch.no_grad():
        for n, p in m.named_parameters():
            if p.dim() >= 2 and "position_embedding" not in n:
                p.normal_(0, (1.0 / p[0].numel()) ** 0.5)
            elif "bias" in n or "class_embedding" in n:
                p.normal_(0, 0.1)
            elif "position_embedding" in n:
                p.normal_(0, 0.5)
    return m


def test_mirror_matches_transformers_over_emulated_kernels():
    from animate_anything_b200.clip_vision import CLIPVisionModelWithProjection
    hf = hf_vision()
    ours = CLIPVisionModelWithProjection.from_hf(hf)
    assert sorted(ours.state_dict()) == sorted(k for k in hf.state_dict() if not k.endswith("position_ids"))
    g = torch.Generator().manual_seed(1)
    pv = torch.randn(2, 3, 224, 224, generator=g)
    with torch.no_grad():
        ref = hf(pixel_values=pv)
    from animate_anything_b200 import ops
    with cve.emulated_vision_ops():
        prep = ours._build_prepared(torch.float32, torch.device("cpu"))
        x = ops.clip_image_prep(pv, torch.float32, 224, 14, ours.k_pad)
        out = ours._tower(prep, x, 2)
    assert ours.k_pad == 592 and x.shape == (2 * 257, 592)
    assert out.image_embeds.shape == ref.image_embeds.shape == (2, 96)
    assert out.last_hidden_state.shape == ref.last_hidden_state.shape == (2, 257, 160)
    assert (out.last_hidden_state - ref.last_hidden_state).abs().max().item() < 5e-4
    assert (out.image_embeds - ref.image_embeds).abs().max().item() < 5e-4


def test_mirror_config_and_refusals(tmp_path):
    from animate_anything_b200.clip_vision import CLIPVisionModelWithProjection
    with pytest.raises(ValueError):
        CLIPVisionModelWithProjection(hidden_size=1024, num_attention_heads=16)           # head dim 64
    with pytest.raises(ValueError):
        CLIPVisionModelWithProjection(**SMALL, hidden_act="relu")
    hf = hf_vision(act="quick_gelu")
    hf.save_pretrained(str(tmp_path / "image_encoder"))
    m = CLIPVisionModelWithProjection.from_pretrained(str(tmp_path), subfolder="image_encoder")
    assert m.config.hidden_act == "quick_gelu" and m.config.projection_dim == 96
    for k, v in hf.state_dict().items():
        if not k.endswith("position_ids"):
            assert torch.equal(m.state_dict()[k], v), k
    with pytest.raises(TypeError):                                   # fp32 on the CPU: no fallback
        m(torch.zeros(1, 3, 224, 224))
    with pytest.raises(ValueError, match=r"Input image size \(576\*1024\) doesn't match model \(224\*224\)"):
        m(torch.zeros(1, 3, 576, 1024))
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 224, 224), output_hidden_states=True)
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 224, 224), interpolate_pos_encoding=True)


# ---------------------------------------------------------------------------------------------- preprocessing pins
def test_blur_restatement_matches_torchvision():
    import torchvision.transforms.functional as TF
    from animate_anything_b200.clip_vision import gaussian_taps
    g = torch.Generator().manual_seed(2)
    x = torch.rand(2, 3, 40, 57, generator=g) * 2 - 1
    for (ky, sy), (kx, sx) in [((3, 0.7857), (7, 1.7857)), ((5, 1.1), (3, 0.001)), ((9, 2.2), (11, 2.7))]:
        got = cve.gaussian_blur_reflect(x, gaussian_taps(ky, sy), gaussian_taps(kx, sx))
        want = TF.gaussian_blur(x, kernel_size=[kx, ky], sigma=[sx, sy])             # reflect padding
        assert (got - want).abs().max().item() < 2e-6, (ky, kx)


def test_resize_restatement_matches_interpolate():
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(3)
    for h, w in [(576, 1024), (333, 577), (80, 100), (224, 224)]:
        x = torch.rand(1, 3, h, w, generator=g) * 2 - 1
        got = cve.bicubic_align_corners(x, (224, 224))
        want = F.interpolate(x, size=(224, 224), mode="bicubic", align_corners=True)
        assert (got - want).abs().max().item() < 2e-6, (h, w)


def test_normalisation_matches_clip_image_processor():
    from transformers import CLIPImageProcessor
    fe = CLIPImageProcessor()
    g = torch.Generator().manual_seed(4)
    u8 = (torch.rand(2, 224, 224, 3, generator=g) * 255).to(torch.uint8)
    unit = u8.permute(0, 3, 1, 2).float() / 255.0
    want = fe(images=unit, do_normalize=True, do_center_crop=False, do_resize=False, do_rescale=False,
              return_tensors="pt").pixel_values
    m = torch.tensor(fe.image_mean, dtype=torch.float32).view(1, 3, 1, 1)
    s = torch.tensor(fe.image_std, dtype=torch.float32).view(1, 3, 1, 1)
    assert torch.equal((unit - m) / s, want)
    assert tuple(fe.image_mean) == pytest.approx(cve.clip_vision.OPENAI_CLIP_MEAN)
    assert tuple(fe.image_std) == pytest.approx(cve.clip_vision.OPENAI_CLIP_STD)


def test_recalled_diffusers_facts():
    """Parity unpinned (diffusers is not in the image): one assertion per recalled fact."""
    from animate_anything_b200.clip_vision import antialias_params, gaussian_taps
    from animate_anything_b200.image_processor import VaeImageProcessor
    # sigma = max((factor - 1) / 2, 0.001), ks = int(max(4 sigma, 3)) bumped to odd
    (ky, sy), (kx, sx) = antialias_params(576, 1024)
    assert (ky, kx) == (3, 7) and sy == pytest.approx((576 / 224 - 1) / 2) and sx == pytest.approx((1024 / 224 - 1) / 2)
    assert antialias_params(80, 100) == ((3, 0.001), (3, 0.001))
    assert antialias_params(1344, 2048)[0][0] == 11 and antialias_params(1120, 224)[0][0] == 9        # 8 -> 9 (odd)
    assert torch.equal(gaussian_taps(3, 0.001), torch.tensor([0.0, 1.0, 0.0]))
    # /255: pil_to_numpy, as the pinned VaeImageProcessor mirror does it
    import PIL.Image
    u8 = (np.arange(48 * 64 * 3) % 256).astype(np.uint8).reshape(48, 64, 3)
    want = torch.from_numpy(VaeImageProcessor.pil_to_numpy(PIL.Image.fromarray(u8))).permute(0, 3, 1, 2)
    assert torch.equal(torch.from_numpy(u8)[None].permute(0, 3, 1, 2).float() / 255.0, want)
    # step order: [-1, 1] around the antialiased resize, then the normaliser; at the model's size the resize is the
    # identity and the sequence equals the CLIP processor's own rescale + normalise
    from transformers import CLIPImageProcessor
    u8 = torch.from_numpy((np.arange(224 * 224 * 3) * 7 % 256).astype(np.uint8).reshape(1, 224, 224, 3))
    got = cve.preprocess_u8(u8)
    want = CLIPImageProcessor()(images=u8.permute(0, 3, 1, 2).float(), do_resize=False, do_center_crop=False,
                                return_tensors="pt").pixel_values
    assert (got - want).abs().max().item() < 1e-5


# ---------------------------------------------------------------------------------------------- C-ABI argument checks
def test_new_entry_points_reject_bad_arguments_without_a_gpu():
    from animate_anything_b200 import _lib
    lib = _lib.load()
    buf = (C.c_float * 4096)()
    p = C.c_void_p((C.addressof(buf) + 15) // 16 * 16)
    mis = C.c_void_p(p.value + 2)

    def fa(q=p, kv=p, out=p, ldq=240, ldkv=240, ld_out=80, nb=1, lq=4, lk=4, heads=1, bf=0, k_col0=80, v_col0=160):
        return lib.aab_flash_attn_d80(q, ldq, lq * ldq, 240, 0, kv, ldkv, lk * ldkv, 240, k_col0, v_col0, out, ld_out,
                                      lq * ld_out, 0, nb, nb, 1, heads, lq, lk, 0.1, bf, None)
    assert fa(q=None) == 1 and fa(kv=None) == 1 and fa(out=None) == 1
    assert fa(lk=0) == 1 and fa(lq=0) == 1 and fa(heads=0) == 1 and fa(nb=0) == 1
    assert fa(ldq=244) == 1 and fa(ld_out=84) == 1                                  # row strides not multiples of 8
    assert fa(q=mis) == 1                                                           # base not 16-byte aligned
    assert fa(bf=2) == 1                                                            # no causal variant
    assert fa(heads=3) == 1 and fa(v_col0=200) == 1                                 # heads past the given columns

    def prep(src=p, st=0, h=8, w=8, ks=3, out=p, out_size=28, patch=14, ld=592, taps=p):
        return lib.aab_clip_image_prep(src, st, h * w * 3, 1, w * 3, 3, 1, h, w, taps, ks, taps, ks, taps, out_size, patch,
                                       out, ld, 0, None)
    assert prep(src=None) == 1 and prep(out=None) == 1 and prep(taps=None) == 1
    assert prep(out_size=30) == 1                                                   # not divisible by the patch
    assert prep(ld=580) == 1 and prep(ld=596) == 1                                  # narrower than 588 / not a multiple of 8
    assert prep(out=mis) == 1
    assert prep(ks=4) == 1 and prep(ks=17) == 1                                     # even taps / reflect pad wider than the image
    assert prep(st=1) == 1                                                          # a float source must be out_size^2
    assert prep(st=5) == 1
