"""Generate tests/golden/long_prompt.npz by running the UNMODIFIED reference functions on a long prompt.

    python tests/golden/make_long_prompt_golden.py     (needs a reference checkout named by PWW_REFERENCE_ROOT)

A long aurora_1 prompt is split into 77-token CLIP chunks by the product's chunker (conditioning.chunk_prompt); the
reference's `_tokens_img_attention_weight` sizes its map by the id count, so it runs unchanged on the concatenated
chunked ids.  The archive holds:

  ids                 the chunked ids [154] (2 chunks)
  w8 .. w64           reference `_tokens_img_attention_weight` at ratios 8/16/32/64 on those ids
  orig_shape/_digest  the same at ratio 1 (ORIG map, [512, 512, 154]): shape and exact digest
  attn.*, x, ctx, w   a CrossAttention module, its input and a [64, 154] weight map (a label in each chunk)
  out_dict_max / _std reference `inj_forward` (CPU fp32) with a 154-token dict context, max and std weight functions

The archive is rewritten only when its arrays change, so re-running leaves it byte-identical.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_loader import REFERENCE_ROOT, load_reference  # noqa: E402
from paint_with_words_sd_b200.conditioning import chunk_prompt  # noqa: E402
from paint_with_words_sd_b200.synthetic import SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import CrossAttention  # noqa: E402
from tests.fixtures import SETTINGS, exact_digest  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "long_prompt.npz")
PNG = "aurora_1.png"

# ~117 tokens: "full moon" sits at prompt tokens 74-75, so a plain 75-token cut would split it; the chunker ends the
# first window before the label instead
LONG_AURORA_PROMPT = (
    "A digital painting of a half-frozen lake near mountains under a full moon and aurora. A boat is in the middle of "
    "the lake. Highly detailed, intricate brush strokes, soft cold light, deep blue and green tones, gentle mist over "
    "the water, reflections of the sky on the ice, quiet northern night, many bright stars scattered across the vast "
    "dark heavens, the full moon glowing, faint snow on the pine trees along the shore, aurora ribbons in the sky, a "
    "small wooden boat, cinematic composition, trending on artstation, sharp focus, volumetric light, calm and serene "
    "atmosphere.")


def build(ref) -> dict:
    tok = SimpleWordTokenizer()
    s = SETTINGS["aurora"]
    lp = {}
    img = Image.open(os.path.join(REFERENCE_ROOT, "contents", PNG)).convert("RGB")
    labels = [v.rpartition(",")[0] for v in s["ctx"].values()]
    ids = chunk_prompt(tok, LONG_AURORA_PROMPT, labels, max_prompt_chunks=3)
    lp["ids"] = ids[0].numpy()
    sep, _, _ = ref._image_context_seperator(img, dict(s["ctx"]), tok)
    text_input = {"input_ids": ids}
    for r in (8, 16, 32, 64):
        lp[f"w{r}"] = ref._tokens_img_attention_weight(sep, text_input, ratio=r).numpy()
    orig = ref._tokens_img_attention_weight(sep, text_input, ratio=1, original_shape=True)
    lp["orig_shape"] = np.array(orig.shape)
    lp["orig_digest"] = exact_digest(orig)

    g = torch.Generator().manual_seed(20261015)
    heads, d, n_side, dc, T = 2, 40, 8, 32, 154
    C, N = heads * d, n_side * n_side
    attn = CrossAttention(C, dc, heads, d)
    for p in attn.parameters():
        p.data = torch.randn(p.shape, generator=g) * (0.3 if p.dim() > 1 else 0.05)
    x = torch.randn(1, N, C, generator=g)
    ctx = torch.randn(1, T, dc, generator=g)
    w = torch.zeros(N, T)
    w[:, 3] = (torch.rand(N, generator=g) > 0.5).float() * 1.5
    w[:, 90:92] = (torch.rand(N, 1, generator=g) > 0.7).float() * 0.4      # a label in the second chunk
    w[:, 140] = (torch.rand(N, generator=g) > 0.4).float() * 0.8
    sigma = torch.tensor(7.25)
    for name, p in attn.named_parameters():
        lp[f"attn.{name}"] = p.detach().numpy()
    lp.update(x=x.numpy(), ctx=ctx.numpy(), w=w.numpy(), sigma=np.float32(sigma.item()), heads=np.int64(heads))
    fns = {"max": lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max(),
           "std": lambda w, sigma, qk: 0.5 * w * math.log(1 + sigma) * qk.std()}
    with torch.no_grad():
        for fname, f in fns.items():
            c = {"CONTEXT_TENSOR": ctx, f"CROSS_ATTENTION_WEIGHT_{N}": w, "CROSS_ATTENTION_WEIGHT_ORIG": 0,
                 "SIGMA": sigma, "WEIGHT_FUNCTION": f}
            lp[f"out_dict_{fname}"] = ref.inj_forward(attn, x, c).numpy()
    return lp


def main():
    arrays = build(load_reference())
    if os.path.exists(OUT):
        with np.load(OUT) as old:
            if set(old.files) == set(arrays) and all(
                    old[k].dtype == np.asarray(v).dtype and np.array_equal(old[k], np.asarray(v)) for k, v in arrays.items()):
                print(OUT, "unchanged")
                return
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
