"""Attention recording without a GPU: the token -> region row against the reference-pinned weight maps
(tests/golden/*.npz), its rules (first region wins, missing labels, long prompts, the 16-region limit), the recording
C entry points' argument checks and the adherence arithmetic."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle.attention_maps import token_regions
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.pipeline import region_adherence, region_coverage
from paint_with_words_sd_b200.synthetic import SimpleWordTokenizer
from tests.fixtures import GOLDEN, SETTINGS, color_map_image
from tests.golden.make_long_prompt_golden import LONG_AURORA_PROMPT

TOK = SimpleWordTokenizer()


def _labels(ctx):
    return [v.rpartition(",")[0] for v in ctx.values()]


def _check_against_golden(row, sep, ids, golden_w):
    """row is the first-region rule applied to the reference's columns: token t has a region iff the reference writes a
    mask into column t, and the region it gets is the first whose label covers t."""
    t = len(ids)
    cols = C._cidx_columns(t)
    assert row.dtype == torch.int8 and row.shape == (C.PACK_TOKENS * C.key_chunks(t),)
    assert (row[[c for c in range(row.numel()) if c not in set(cols.tolist())]] == -1).all()
    got = row[cols].tolist()
    written = (torch.from_numpy(golden_w) != 0).any(0).tolist()
    assert [g >= 0 for g in got] == written
    owner = token_regions([lab for lab, _ in sep], ids)
    assert got == owner
    # each owner's resized mask is part of what the reference added into the column
    ratio = 8
    for tok, r in enumerate(got):
        if r >= 0:
            dim0, dim1 = sep[r][1].shape
            m = C._img_importance_flatten(sep[r][1], C.always_round(dim0 / ratio), C.always_round(dim1 / ratio))
            assert (torch.from_numpy(golden_w[:, tok]) >= m.reshape(-1) - 1e-6).all()


@pytest.mark.parametrize("name", ["cat_dog", "aurora"])
def test_region_token_index_against_reference_maps(name):
    g = np.load(os.path.join(GOLDEN, "mask_builder.npz"))
    s = SETTINGS[name]
    sep, _, _ = C._image_context_seperator(color_map_image(name, 512), dict(s["ctx"]), TOK)
    ids = g[f"{name}_512_ids"].tolist()
    assert (g[f"{name}_512_region_pixels"] > 0).all()
    row = C.region_token_index(sep, {"input_ids": torch.tensor([ids])})
    _check_against_golden(row, sep, ids, g[f"{name}_512_w8"])


def test_region_token_index_two_chunks_against_reference_maps():
    g = np.load(os.path.join(GOLDEN, "long_prompt.npz"))
    s = SETTINGS["aurora"]
    ids = C.chunk_prompt(TOK, LONG_AURORA_PROMPT, _labels(s["ctx"]), 3)
    assert ids.shape[1] == 154 and ids[0].tolist() == g["ids"].tolist()
    sep, _, _ = C._image_context_seperator(color_map_image("aurora", 512), dict(s["ctx"]), TOK)
    row = C.region_token_index(sep, {"input_ids": ids})
    _check_against_golden(row, sep, ids[0].tolist(), g["w8"])
    assert row.shape == (160,) and (row[77:80] == -1).all() and (row[157:] == -1).all()


def test_region_token_index_three_chunks():
    s = SETTINGS["aurora"]
    prompt = " ".join([LONG_AURORA_PROMPT, s["prompt"], s["prompt"]])
    ids = C.chunk_prompt(TOK, prompt, _labels(s["ctx"]), 3)
    assert ids.shape[1] == 231
    sep, _, _ = C._image_context_seperator(color_map_image("aurora", 128), dict(s["ctx"]), TOK)
    row = C.region_token_index(sep, {"input_ids": ids})
    w = C._tokens_img_attention_weight(sep, {"input_ids": ids}, ratio=8)
    _check_against_golden(row, sep, ids[0].tolist(), w.numpy())
    assert row.shape == (240,) and all((row[80 * c + 77:80 * c + 80] == -1).all() for c in range(3))
    assert all((row[80 * c:80 * c + 77] >= 0).any() for c in range(3))     # every chunk holds painted words


def _sep(ctx, prompt, size=64):
    """Regions of a colour map with one horizontal band per colour."""
    img = np.zeros((size, size, 3), dtype=np.uint8)
    for i, c in enumerate(ctx):
        img[i * size // len(ctx):(i + 1) * size // len(ctx)] = c
    sep, _, _ = C._image_context_seperator(Image.fromarray(img), dict(ctx), TOK)
    ids = TOK([prompt], padding="max_length", max_length=TOK.model_max_length, truncation=True,
              return_tensors="pt")["input_ids"]
    return sep, ids


def test_repeated_label_gives_every_span_the_region():
    sep, ids = _sep({(0, 0, 0): "cat,1.0", (255, 255, 255): "dog,1.0"}, "a cat and a dog and another cat")
    row = C.region_token_index(sep, {"input_ids": ids})
    toks = ids[0].tolist()
    cat, dog = TOK("cat")["input_ids"][1], TOK("dog")["input_ids"][1]
    assert [row[t].item() for t, i in enumerate(toks) if i == cat] == [0, 0]
    assert [row[t].item() for t, i in enumerate(toks) if i == dog] == [1]
    assert int((row >= 0).sum()) == 3


@pytest.mark.parametrize("moon_first", [True, False])
def test_overlapping_labels_go_to_the_first_region(moon_first):
    items = [((1, 1, 1), "moon,1.0"), ((2, 2, 2), "full moon,1.0")]
    ctx = dict(items if moon_first else items[::-1])
    sep, ids = _sep(ctx, "a full moon over a lake")
    row = C.region_token_index(sep, {"input_ids": ids})
    toks = ids[0].tolist()
    full, moon = toks.index(TOK("full")["input_ids"][1]), toks.index(TOK("moon")["input_ids"][1])
    moon_slot, full_slot = (0, 1) if moon_first else (1, 0)
    assert row[full].item() == full_slot
    assert row[moon].item() == (moon_slot if moon_first else full_slot)


def test_missing_label_gets_no_tokens():
    sep, ids = _sep({(0, 0, 0): "zebra,1.0", (255, 255, 255): "lake,1.0"}, "a calm lake")
    row = C.region_token_index(sep, {"input_ids": ids})
    assert not (row == 0).any() and int((row == 1).sum()) == 1


def test_more_than_16_regions_raise():
    ctx = {(i, i, i): f"w{i},1.0" for i in range(17)}
    sep, ids = _sep(ctx, " ".join(f"w{i}" for i in range(17)), size=68)
    with pytest.raises(ValueError, match="16 regions"):
        C.region_token_index(sep, {"input_ids": ids})
    assert C.region_token_index(sep[:16], {"input_ids": ids}).max().item() == 15


def test_conditioning_builder_carries_the_row():
    s = SETTINGS["aurora"]
    from paint_with_words_sd_b200.synthetic import RandomTextEncoder
    _, sep, cond, uncond = C._encode_text_color_inputs(RandomTextEncoder(64), TOK, "cpu", color_map_image("aurora", 128),
                                                       dict(s["ctx"]), s["prompt"], "")
    assert cond[C.REGION_COUNT_KEY] == 5
    assert torch.equal(cond[C.REGION_INDEX_KEY], C.region_token_index(sep, TOK([s["prompt"]], padding="max_length",
                                                                                max_length=77, truncation=True,
                                                                                return_tensors="pt")))
    assert C.REGION_INDEX_KEY not in uncond


# ---- the C entry points' argument checks (before any CUDA call) ----
def _rec_call(L, ridx, rec_index, rec_acc, rec_bs, B=2, H=8, N=64, T=77, D=40):
    buf = (ctypes.c_char * 8192)()
    p16 = (ctypes.addressof(buf) + 15) // 16 * 16
    C_ = H * D
    return L(p16, p16, p16, p16, B, H, N, T, D, N * C_, C_, T * C_, C_, N * C_, C_, None, 0, 0, None, None, None,
             None, 0.158, None, None, 0, None, ridx, rec_index, rec_acc, rec_bs), p16


@pytest.mark.parametrize("suffix", ["f16", "bf16"])
def test_rec_entry_rejects_bad_arguments(suffix):
    L = getattr(_native.lib(), f"pww_xattn_fused_rec_{suffix}")
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    ok_bs = 8 * 64 * 16
    assert _rec_call(L, None, a, a, ok_bs)[0] == -1                 # null ridx
    assert _rec_call(L, a, None, a, ok_bs)[0] == -1                 # null rec_index
    assert _rec_call(L, a, a, None, ok_bs)[0] == -1                 # null rec_acc
    assert _rec_call(L, a, a, a + 4, ok_bs)[0] == -1                # rec_acc not 16-byte aligned
    assert _rec_call(L, a, a, a, ok_bs - 1)[0] == -1                # records overlap
    # the _multi checks still come first: an unsupported head dim is reported as such
    assert _rec_call(L, a, a, a, ok_bs, D=48)[0] == -2


def test_rec_entry_is_declared_with_the_multi_arguments_plus_four():
    L = _native.lib()
    for s in ("f16", "bf16"):
        rec, multi = getattr(L, f"pww_xattn_fused_rec_{s}"), getattr(L, f"pww_xattn_fused_multi_{s}")
        assert list(rec.argtypes[:-4]) == list(multi.argtypes) and len(rec.argtypes) == len(multi.argtypes) + 4


# ---- adherence ----
def test_adherence_arithmetic():
    maps = torch.zeros(3, 4, 4)
    maps[0, :2] = 1.0                      # all of region 0's attention in the top half
    maps[1] = 1.0                          # region 1 attends everywhere
    cov = torch.zeros(3, 4, 4)
    cov[0, :2] = 1.0
    cov[1, :, :1] = 0.5                    # region 1 covers half of the first column
    cov[2] = 1.0
    adh = region_adherence(maps, cov, [True, True, False])
    assert adh.dtype == torch.float32
    assert adh[0].item() == 1.0
    assert math.isclose(adh[1].item(), (4 * 0.5) / 16)
    assert math.isnan(adh[2].item())


def test_coverage_is_the_area_fraction_of_the_binary_mask():
    img = np.zeros((16, 16, 3), dtype=np.uint8)
    img[:, :4] = (255, 0, 0)               # the left quarter
    img[0, 0] = (0, 255, 0)                # one pixel of another colour
    cov = region_coverage(Image.fromarray(img), {(255, 0, 0): "a,1", (0, 255, 0): "b,1", (0, 0, 9): "c,1"}, (2, 2))
    assert cov.shape == (3, 2, 2)
    assert torch.allclose(cov[0], torch.tensor([[0.5 - 1 / 64, 0.0], [0.5, 0.0]]))
    assert math.isclose(cov[1].sum().item(), 1 / 64) and cov[2].sum().item() == 0.0
