"""Negative region prompts on the CPU: the shared chunk layout and both sides' ids and weights, the statistic-chunk
masks, every argument error, batch grouping, the new C entry points, and the oracle's fp64 self-checks."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import negative_region as NO
from oracle import pww_oracle as O
from oracle import region_prompt as RO
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from tests.fixtures import SETTINGS, color_map_image

TOK = SimpleWordTokenizer()
RED, BLUE, GREEN = (255, 0, 0), (0, 0, 255), (0, 255, 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("pww_xattn_fused_region_rows_f16", "pww_xattn_fused_region_rows_bf16",
               "pww_xattn_fused_region_rows_multi_f16", "pww_xattn_fused_region_rows_multi_bf16")


def _two_region_map(h, w):
    a = np.zeros((h, w, 3), dtype=np.uint8)
    a[:, : w // 3] = RED
    a[h // 2:, w // 2:] = BLUE
    return Image.fromarray(a)


def _encode(region_prompts=None, negative=None, beta=0.2, uncond="", img=None, **kw):
    s = SETTINGS["cat_dog"]
    img = color_map_image("cat_dog", 128) if img is None else img
    return C._encode_text_color_inputs(RandomTextEncoder(32), TOK, "cpu", img, dict(s["ctx"]), s["prompt"], uncond,
                                       region_prompts=region_prompts, region_base_ratio=beta,
                                       negative_region_prompts=negative, **kw)


def _chunk_words(ids, c):
    bos, eos, pad = C._special_ids(TOK, 77)
    chunk = ids[0, 77 * c: 77 * (c + 1)].tolist()
    assert chunk[0] == bos
    end = chunk.index(eos)
    assert chunk[end + 1:] == [pad] * (76 - end)
    return chunk[1:end]


def _words(text):
    return list(TOK(text)["input_ids"])[1:-1]


@pytest.mark.parametrize("pos,neg,layout", [
    ({RED: "a"}, None, [RED]),
    (None, {BLUE: "b"}, [BLUE]),
    ({RED: "a"}, {BLUE: "b"}, [RED, BLUE]),
    ({RED: "a", BLUE: "b"}, {"#0000ff": "c"}, [RED, BLUE]),          # one colour in two key forms
    ({BLUE: "b"}, {RED: "c", "#0000ff": "d"}, [BLUE, RED]),
])
def test_layout_orders_positive_then_negative_colours(pos, neg, layout):
    assert C.region_layout(pos, neg) == layout


def test_chunk_ids_of_both_sides():
    ctx = SETTINGS["cat_dog"]["ctx"]
    a, b = list(ctx)[:2]
    base = SETTINGS["cat_dog"]["prompt"]
    cases = [
        # positives, negatives -> cond sentences per chunk, uncond sentences per chunk (None: today's uncond windows)
        ({a: "red lantern"}, None, ["red lantern"], None),
        (None, {b: "blurry trees"}, [base], ["blurry trees"]),
        ({a: "red lantern"}, {b: "blurry trees"}, ["red lantern", base], ["ugly", "blurry trees"]),
        ({a: "red lantern", b: "green tree"}, {a: "dark"}, ["red lantern", "green tree"], ["dark", "ugly"]),
    ]
    for pos, neg, cond_texts, un_texts in cases:
        uncond = "ugly"
        layout = C.region_layout(pos, neg)
        texts, bits = C._side_sentences(layout, pos, base)
        ids = C.region_chunk_ids(TOK, base, texts)
        assert ids.shape == (1, 77 * (1 + len(layout)))
        assert [_chunk_words(ids, c) for c in range(1 + len(layout))] == [_words(t) for t in [base] + cond_texts]
        assert bits == sum(1 << c for c, col in enumerate(layout, 1) if pos and col in pos)
        if un_texts is not None:
            texts, bits = C._side_sentences(layout, neg, uncond)
            ids = C.region_chunk_ids(TOK, uncond, texts)
            assert [_chunk_words(ids, c) for c in range(1 + len(layout))] == [_words(t) for t in [uncond] + un_texts]
            assert bits == sum(1 << c for c, col in enumerate(layout, 1) if col in neg)


def test_dicts_carry_both_sides_and_their_sentence_masks():
    ctx = SETTINGS["cat_dog"]["ctx"]
    a, b = list(ctx)[:2]
    _, _, cond, uncond = _encode({a: "a red thing"}, {b: "a blue thing"}, uncond="blurry")
    assert cond[C.REGION_SENTENCES_KEY] == 0b010 and uncond[C.REGION_SENTENCES_KEY] == 0b100
    assert cond["CONTEXT_TENSOR"].shape[1] == 231 and uncond["CONTEXT_TENSOR"].shape[1] == 231
    enc = RandomTextEncoder(32)
    un = uncond["CONTEXT_TENSOR"]
    blurry = enc(C._chunked_ids(TOK, [_words("blurry")], 1))[0]
    assert torch.equal(un[:, :77], blurry) and torch.equal(un[:, 77:154], blurry)   # chunk 1: the uncond prompt again
    assert torch.equal(un[:, 154:], enc(C._chunked_ids(TOK, [_words("a blue thing")], 1))[0])
    for n in (256, 64, 16, 4):
        wc, wu = cond[C.region_key(n)], uncond[C.region_key(n)]
        assert not wc[:, 2].any() and not wu[:, 1].any()        # each side weighs only its own sentences
    assert cond[C.region_key(256)][:, 1].any() and uncond[C.region_key(256)][:, 2].any()
    # negative-only: the cond side is the plain call's chunk 0 everywhere
    _, _, cond, uncond = _encode(None, {b: "a blue thing"})
    assert cond[C.REGION_SENTENCES_KEY] == 0 and uncond[C.REGION_SENTENCES_KEY] == 0b10
    for n in (256, 64, 16, 4):
        assert torch.equal(cond[C.region_key(n)][:, 0], torch.ones(n)) and not cond[C.region_key(n)][:, 1:].any()


@pytest.mark.parametrize("beta", [0.0, 0.2, 0.7, 1.0])
def test_each_sides_weights_are_convex_and_base_only_outside_its_regions(beta):
    img = _two_region_map(128, 192)
    pixels = np.array(img)
    layout = C.region_layout({RED: "a"}, {BLUE: "b", GREEN: "absent"})
    for side in ({RED: "a"}, {BLUE: "b", GREEN: "absent"}):
        for r in C.RATIOS:
            w = C.region_chunk_weights(img, side, beta, r, layout)
            assert w.dtype == torch.float32 and w.shape[1] == 1 + len(layout)
            assert (w >= 0).all() and (w <= 1).all()
            assert torch.allclose(w.sum(1), torch.ones(w.shape[0]), atol=1e-6)
            r0, r1 = C.always_round(128 / r), C.always_round(192 / r)
            inside = torch.zeros(r0 * r1, dtype=torch.bool)
            for c, colour in enumerate(layout, start=1):
                if colour not in side:
                    assert not w[:, c].any()
                    continue
                f = O.img_importance_flatten(torch.from_numpy((pixels == colour).all(-1)).float(), r0, r1).reshape(-1)
                assert torch.equal(w[:, c], (1 - beta) * f)
                inside |= f > 0
            assert torch.equal(w[~inside, 0], torch.ones(int((~inside).sum())))


def _same_dict(x, y):
    assert sorted(x) == sorted(y)
    for k in x:
        if isinstance(x[k], torch.Tensor):
            assert torch.equal(x[k], y[k]), k
        else:
            assert x[k] == y[k], k


@pytest.mark.parametrize("which", ["same", "one", "other_key_form"])
def test_cond_dict_is_the_region_only_calls_when_negatives_share_its_colours(which):
    ctx = SETTINGS["cat_dog"]["ctx"]
    a, b = list(ctx)[:2]
    pos = {a: "a small red lantern", b: "a tall green tree"}
    neg = {"same": {a: "blurry", b: "ugly"}, "one": {b: "ugly"},
           "other_key_form": {"#%02x%02x%02x" % b: "ugly"}}[which]
    _, _, ref, ref_un = _encode(pos, uncond="bad")
    _, _, got, got_un = _encode(pos, neg, uncond="bad")
    _same_dict(got, ref)
    assert got_un[C.REGION_SENTENCES_KEY] != 0 and ref_un[C.REGION_SENTENCES_KEY] == 0


def test_region_only_calls_keep_their_uncond_side():
    _, _, cond, uncond = _encode({RED: "a"}, uncond="bad")
    assert uncond[C.REGION_SENTENCES_KEY] == 0 and cond[C.REGION_SENTENCES_KEY] == 0b10
    for n in (256, 64, 16, 4):
        assert torch.equal(uncond[C.region_key(n)][:, 0], torch.ones(n)) and not uncond[C.region_key(n)][:, 1:].any()


@pytest.mark.parametrize("kwargs,match", [
    (dict(region_prompts={RED: "a"}, negative={BLUE: "b", GREEN: "c"}), "3 colours in all"),
    (dict(negative={RED: "a", BLUE: "b", GREEN: "c"}), "3 colours in all"),
    (dict(negative={}), "negative_region_prompts takes"),
    (dict(negative={RED: "a"}, max_prompt_chunks=2), "max_prompt_chunks"),
    (dict(region_prompts={RED: "a"}, negative={RED: "b"}, max_prompt_chunks=3), "max_prompt_chunks"),
    (dict(negative={RED: "a"}, beta=1.5), r"\[0, 1\]"),
    (dict(negative={RED: "a"}, beta=-0.1), r"\[0, 1\]"),
    (dict(negative={RED: " ".join(["word"] * 76)}), "negative region prompt .* 75-token"),
    (dict(negative={RED: "a"}, uncond=" ".join(["word"] * 76)), "unconditional_input_prompt .* 75-token"),
    (dict(region_prompts={RED: " ".join(["word"] * 76)}, negative={RED: "a"}), "region prompt .* 75-token"),
    (dict(negative={RED: "a"}, img=_two_region_map(96, 128)), "multiples of 64"),
])
def test_negative_region_argument_errors(kwargs, match):
    kw = dict(kwargs)
    with pytest.raises(ValueError, match=match):
        _encode(kw.pop("region_prompts", None), kw.pop("negative"), **kw)


def test_negative_regions_need_a_colour_map():
    with pytest.raises(ValueError, match="color_map_image"):
        C._encode_text_color_inputs(RandomTextEncoder(32), TOK, "cpu", None, {}, "x", "",
                                    negative_region_prompts={RED: "a"})


def test_check_needs_no_model():
    C.check_negative_region_prompts({RED: "a", BLUE: "b"}, {"#ff0000": "c"}, 0.2)
    C.check_negative_region_prompts(None, {RED: "c"}, 0.0, 1)
    with pytest.raises(ValueError, match="3 colours"):
        C.check_negative_region_prompts({RED: "a", BLUE: "b"}, {GREEN: "c"}, 0.2)
    with pytest.raises(ValueError, match="1 .. 2"):
        C.check_negative_region_prompts({RED: "a", BLUE: "b", GREEN: "c"}, {RED: "c"}, 0.2)


def test_public_functions_reject_negative_regions_they_cannot_run():
    img = color_map_image("cat_dog", 128)
    with pytest.raises(ValueError, match="attention recording"):
        PL.paint_with_words({RED: "x,1"}, img, "x", negative_region_prompts={RED: "a"}, return_attention_maps=True)
    with pytest.raises(ValueError, match="3 colours"):
        PL.paint_with_words({RED: "x,1"}, img, "x", region_prompts={RED: "a"},
                            negative_region_prompts={BLUE: "b", GREEN: "c"})
    with pytest.raises(ValueError, match="max_prompt_chunks"):
        PL.paint_with_words_inpaint({RED: "x,1"}, img, img, img, "x", negative_region_prompts={RED: "a"},
                                    max_prompt_chunks=3)
    with pytest.raises(ValueError, match=r"settings\[1\]: .*\[0, 1\]"):
        PL.paint_with_words_batch([dict(color_map_image=img),
                                   dict(color_map_image=img, negative_region_prompts={RED: "a"},
                                        region_base_ratio=2.0)])
    with pytest.raises(ValueError, match=r"settings\[0\]: .*3 colours"):
        PL.paint_with_words_batch([dict(color_map_image=img, region_prompts={RED: "a"},
                                        negative_region_prompts={BLUE: "b", GREEN: "c"})])
    with pytest.raises(ValueError, match="attention recording"):
        PL.paint_with_words_batch([dict(color_map_image=img, negative_region_prompts={RED: "a"})],
                                  return_attention_maps=True)


def test_batch_entries_with_a_sentence_on_either_side_group_together():
    entries = [dict(region_prompts=None, negative_region_prompts=None),
               dict(region_prompts={RED: "a"}, negative_region_prompts=None),
               dict(region_prompts=None, negative_region_prompts={RED: "b"}),
               dict(region_prompts={RED: "a"}, negative_region_prompts={RED: "b"})]
    flags = [PL._has_region_sentence(e) for e in entries]
    assert flags == [False, True, True, True]
    keys = [(8, 8, 154 if f else 77, f) for f in flags]
    assert PL.batch_groups(keys, 8) == [[0], [1, 2, 3]]
    assert "negative_region_prompts" in PL.BATCH_SETTING_KEYS


def test_new_symbols_are_declared_and_exported():
    src = open(os.path.join(ROOT, "include", "pww_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    for name in NEW_SYMBOLS:
        assert re.search(rf"\b{name}\s*\(", src), name
        assert name in _native.EXPORTS


def test_new_entry_points_check_their_arguments():
    L = _native.lib()
    buf = (ctypes.c_char * 4096)()
    p16 = (ctypes.addressof(buf) + 15) // 16 * 16
    for name, stat in zip(NEW_SYMBOLS, (0, 0, None, None)):
        fn = getattr(L, name)

        def call(T, w, ws, q=p16):
            return fn(q, p16, p16, p16, 1, 8, 64, T, 40, 20480, 320, T * 320, 320, 20480, 320, None, 0, 0, None, None,
                      stat, None, 0.158, None, None, 0, None, w, ws, p16, None)
        assert call(77, p16, 64 * 3) == -2                        # one chunk: no region mode
        assert call(154, None, 64 * 2) == -1                      # no weights
        assert call(154, p16 + 2, 64 * 2) == -1                   # misaligned weights
        assert call(231, p16, 64 * 3 - 1) == -1                   # stride below N * k
        assert call(154, p16, 64 * 2, q=None) == -1


# ---------------------------------------------------------------------------------------------------------------
# the oracle, in fp64
# ---------------------------------------------------------------------------------------------------------------
def _qkv(seed, n, t, h, d):
    g = torch.Generator().manual_seed(seed)
    return tuple(torch.randn(1, r, h * d, generator=g, dtype=torch.float64) for r in (n, t, t))


@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("kc", [2, 3])
def test_oracle_statistic_of_chunk_zero_alone_is_the_plain_biased_attention(stat, kc):
    N, H, D = 29, 2, 8
    q, k, v = _qkv(10 + kc, N, 77 * kc, H, D)
    g = torch.Generator().manual_seed(1)
    wmap = (torch.rand(N, 77 * kc, generator=g, dtype=torch.float64) > 0.7).double() * 1.3

    def f(w, sigma, qk):
        return 0.4 * w * (qk.max() if stat == "max" else qk.std())
    weights = torch.zeros(N, kc, dtype=torch.float64)
    weights[:, 0] = 1.0
    got = RO.region_attention_core(q, k, v, H, D ** -0.5, weights,
                                   lambda s: NO.masked_weight_function(f, 0, 77 * kc)(wmap, 1.0, s),
                                   dtype=torch.float64)
    ref = RO.region_attention_core(q, k[:, :77], v[:, :77], H, D ** -0.5, None, lambda s: f(wmap[:, :77], 1.0, s),
                                   dtype=torch.float64)                # one chunk of 77 keys: the plain attention
    assert (got - ref).abs().max().item() < 1e-12
    # and the full mask is the region oracle's statistic over every chunk
    full = RO.region_attention_core(q, k, v, H, D ** -0.5, weights, lambda s: f(wmap, 1.0, s), dtype=torch.float64)
    masked = RO.region_attention_core(q, k, v, H, D ** -0.5, weights,
                                      lambda s: NO.masked_weight_function(f, (1 << kc) - 2, 77 * kc)(wmap, 1.0, s),
                                      dtype=torch.float64)
    assert torch.equal(full, masked)


def test_oracle_negative_sentence_equal_to_the_uncond_prompt_changes_nothing():
    """Every uncond chunk is the uncond prompt's encoding, so any convex weights give its one softmax."""
    a = list(SETTINGS["cat_dog"]["ctx"])[1]
    _, _, _, uncond = _encode(None, {a: "blurry"}, uncond="blurry")
    ctx = uncond["CONTEXT_TENSOR"].double()
    assert torch.equal(ctx[:, :77], ctx[:, 77:])
    N, H, D = 64, 2, 16
    g = torch.Generator().manual_seed(2)
    q = torch.randn(1, N, H * D, generator=g, dtype=torch.float64)
    wk = torch.randn(32, H * D, generator=g, dtype=torch.float64)
    wv = torch.randn(32, H * D, generator=g, dtype=torch.float64)
    k, v = ctx @ wk, ctx @ wv
    w = uncond[C.region_key(N)].double()
    assert w[:, 1].any() and w[:, 0].min() < 1
    got = RO.region_attention_core(q, k, v, H, D ** -0.5, w, dtype=torch.float64)
    ref = RO.region_attention_core(q, k[:, :77], v[:, :77], H, D ** -0.5, None, dtype=torch.float64)
    assert (got - ref).abs().max().item() < 1e-12
