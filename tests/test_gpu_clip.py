"""GPU parity of the CLIP text tower (clip_text.CLIPTextModel on the sm_90a kernels) against the REAL third-party
implementation the reference imports (`transformers.CLIPTextModel`, train.py:88; installed in the image) — this leg of the
path is pinned to the library itself, not to a restatement.  Reference call site: models/pipeline.py:136."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from util import assert_vs_stock, record_parity  # noqa: E402

pytestmark = pytest.mark.gpu


def _hf(layers, hidden, heads, act, seed=0, vocab=1000):
    from transformers import CLIPTextConfig, CLIPTextModel
    torch.manual_seed(seed)
    cfg = CLIPTextConfig(vocab_size=vocab, hidden_size=hidden, intermediate_size=4 * hidden, num_hidden_layers=layers,
                         num_attention_heads=heads, max_position_embeddings=77, hidden_act=act, eos_token_id=vocab - 1,
                         bos_token_id=vocab - 2, pad_token_id=1)
    m = CLIPTextModel(cfg).eval()
    with torch.no_grad():                      # default init is tiny (std 0.02): make the layers matter
        for n, p in m.named_parameters():
            if p.dim() == 2 and "embedding" not in n:
                p.normal_(0, (1.0 / p.shape[1]) ** 0.5)
            elif "bias" in n:
                p.normal_(0, 0.1)
    return m


def _ids(b, vocab, seed=3):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, vocab - 2, (b, 77), generator=g)
    ids[:, 0] = vocab - 2
    for i in range(b):                          # EOS somewhere, padded with EOS after it (CLIP tokenizer behaviour)
        e = 5 + 9 * i
        ids[i, e:] = vocab - 1
    return ids


@pytest.mark.parametrize("dtype,act,layers,hidden,heads", [
    (torch.float16, "gelu", 3, 128, 2),
    (torch.bfloat16, "quick_gelu", 2, 256, 4),
    (torch.float16, "gelu", 23, 1024, 16),      # the ModelScope text tower (OpenCLIP ViT-H/14, penultimate layer), full size
])
def test_clip_text_matches_transformers(dtype, act, layers, hidden, heads):
    from animate_anything_b200.clip_text import CLIPTextModel
    torch.backends.cuda.matmul.allow_tf32 = False
    hf = _hf(layers, hidden, heads, act)
    sd16 = {k: v.to(dtype) for k, v in hf.state_dict().items()}
    hf.load_state_dict({k: v.float() for k, v in sd16.items()})
    ours = CLIPTextModel.from_hf(hf).to(dtype).cuda()
    assert sorted(k for k in ours.state_dict()) == sorted(k for k in hf.state_dict() if not k.endswith("position_ids"))
    ids = _ids(3, hf.config.vocab_size).cuda()
    hf = hf.cuda()
    with torch.no_grad():
        ref = hf(ids)
        stock = hf.to(dtype)(ids)
    out = ours(ids)
    torch.cuda.synchronize()
    assert out[0].shape == ref[0].shape and out.pooler_output.shape == ref.pooler_output.shape
    case = f"CLIP text {layers}L x {hidden} {str(dtype).split('.')[-1]} {act}"
    assert_vs_stock(record_parity(case, "last_hidden_state", out[0], ref[0], stock[0]), max_factor=2.5)
    assert_vs_stock(record_parity(case, "pooler_output", out.pooler_output, ref.pooler_output, stock.pooler_output),
                    max_factor=2.5)


def test_pipeline_prompt_strings_run_on_the_kernels(monkeypatch):
    """`pipe(prompt="...")` with a transformers CLIPTextModel handed in (as train.py:799 does): the pipeline mirrors it
    onto the sm_90a kernels; the library module's forward must never run."""
    from animate_anything_b200.pipeline import LatentToVideoPipeline

    class Tok:
        model_max_length = 77

        def __call__(self, texts, **kw):
            class R:
                pass
            r = R()
            r.input_ids = torch.stack([_ids(1, 1000, seed=len(t))[0] for t in texts])
            return r
    hf = _hf(2, 128, 2, "gelu").half().cuda()

    class FakeUnet:
        dtype = torch.float16
    pipe = LatentToVideoPipeline(vae=None, text_encoder=hf, tokenizer=Tok(), unet=FakeUnet(), scheduler=None)
    with torch.no_grad():
        want = torch.cat([hf(Tok()([""]).input_ids.cuda())[0], hf(Tok()(["a cat"]).input_ids.cuda())[0]]).float()

    def boom(*a, **k):
        raise AssertionError("library CLIP forward was called")
    monkeypatch.setattr(type(hf), "forward", boom)
    got = pipe._encode_prompt("a cat", torch.device("cuda"), 1, True)
    assert got.shape == (2, 77, 128)
    assert (got.float() - want).abs().max().item() <= 2e-2 * want.abs().mean().item() + 2e-2
