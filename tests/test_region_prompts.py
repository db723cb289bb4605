"""Region prompts on the CPU: chunk weights, chunk layout and ids, the argument errors, the C entry points' checks and
the oracle's self-consistency."""
import ctypes

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import pww_oracle as O
from oracle import region_prompt as RO
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from tests.fixtures import SETTINGS, color_map_image

TOK = SimpleWordTokenizer()
RED, BLUE, GREEN = (255, 0, 0), (0, 0, 255), (0, 255, 0)


def _two_region_map(h, w):
    a = np.zeros((h, w, 3), dtype=np.uint8)
    a[:, : w // 3] = RED
    a[h // 2:, w // 2:] = BLUE
    return Image.fromarray(a)


@pytest.mark.parametrize("beta", [0.0, 0.2, 0.7, 1.0])
def test_weights_are_convex_and_sum_to_one(beta):
    img = _two_region_map(128, 192)
    for r in C.RATIOS:
        w = C.region_chunk_weights(img, {RED: "a", BLUE: "b"}, beta, r)
        assert w.dtype == torch.float32 and w.shape[1] == 3
        assert (w >= 0).all() and (w <= 1).all()
        assert torch.allclose(w.sum(1), torch.ones(w.shape[0]), atol=1e-6)
        if beta == 1.0:
            assert torch.equal(w[:, 0], torch.ones(w.shape[0])) and not w[:, 1:].any()


def test_uncovered_pixels_and_absent_colours_get_the_base_prompt_alone():
    img = _two_region_map(128, 128)
    w = C.region_chunk_weights(img, {RED: "a", GREEN: "absent"}, 0.2, 8)
    f_red = C._img_importance_flatten(torch.from_numpy((np.array(img) == RED).all(-1)).float(), 16, 16).reshape(-1)
    far = f_red == 0
    assert far.any()
    assert torch.equal(w[far, 0], torch.ones(int(far.sum()))) and not w[far, 1:].any()
    assert not w[:, 2].any()                                   # green is not in the map


@pytest.mark.parametrize("h,w", [(128, 128), (200, 136), (72, 328)])
def test_weights_follow_the_weight_map_resize_at_every_level(h, w):
    img = _two_region_map(h, w)
    beta = 0.3
    wt = {r: C.region_chunk_weights(img, {"#ff0000": "a", BLUE: "b"}, beta, r) for r in C.RATIOS}
    pixels = np.array(img)
    for r in C.RATIOS:
        r0, r1 = C.always_round(h / r), C.always_round(w / r)
        assert wt[r].shape == (r0 * r1, 3)
        for c, rgb in enumerate((RED, BLUE), start=1):
            mask = torch.from_numpy((pixels == rgb).all(-1)).float()
            f = O.img_importance_flatten(mask, r0, r1).reshape(-1)
            assert torch.equal(wt[r][:, c], (1 - beta) * f)
        assert torch.equal(wt[r][:, 0], 1 - wt[r][:, 1:].sum(1))


def test_chunk_layout_and_ids():
    ids = C.region_chunk_ids(TOK, "a cat and a dog", {RED: "fluffy orange cat", BLUE: "small brown dog"})
    assert ids.shape == (1, 231)
    bos, eos, pad = C._special_ids(TOK, 77)
    for c, text in enumerate(["a cat and a dog", "fluffy orange cat", "small brown dog"]):
        chunk = ids[0, 77 * c: 77 * (c + 1)].tolist()
        words = list(TOK(text)["input_ids"])[1:-1]
        assert chunk == [bos] + words + [eos] + [pad] * (75 - len(words))


def _encode(region_prompts, beta=0.2, size=128, **kw):
    s = SETTINGS["cat_dog"]
    img = color_map_image("cat_dog", size)
    return C._encode_text_color_inputs(RandomTextEncoder(32), TOK, "cpu", img, dict(s["ctx"]), s["prompt"], "",
                                       region_prompts=region_prompts, region_base_ratio=beta, **kw)


def test_dicts_carry_chunked_contexts_and_weights():
    ctx = SETTINGS["cat_dog"]["ctx"]
    colours = list(ctx)[:2]
    _, _, cond, uncond = _encode({colours[0]: "a red thing", colours[1]: "a blue thing"})
    assert cond["CONTEXT_TENSOR"].shape[1] == 231 and uncond["CONTEXT_TENSOR"].shape[1] == 231
    keys = sorted(k for k in cond if k.startswith("REGION_WEIGHTS_"))
    assert keys == sorted(C.region_key(n) for n in (256, 64, 16, 4))
    for k in keys:
        n = int(k.rsplit("_", 1)[1])
        assert cond[k].shape == (n, 3) and cond[C.weight_key(n)].shape == (n, 231)
        assert torch.equal(uncond[k][:, 0], torch.ones(n)) and not uncond[k][:, 1:].any()
    # the uncond prompt is encoded to the same chunks: [BOS, EOS, pad ..] each, the long-prompt layout
    enc = RandomTextEncoder(32)
    one = enc(C._chunked_ids(TOK, [], 1))[0]
    assert torch.equal(uncond["CONTEXT_TENSOR"][:, :77], one) and torch.equal(uncond["CONTEXT_TENSOR"][:, 77:154], one)


def test_plain_calls_have_no_region_keys():
    _, _, cond, uncond = _encode(None)
    assert not any(k.startswith("REGION_WEIGHTS_") for k in list(cond) + list(uncond))


@pytest.mark.parametrize("kwargs,match", [
    (dict(region_prompts={RED: "a"}, max_prompt_chunks=2), "max_prompt_chunks"),
    (dict(region_prompts={RED: "a", BLUE: "b", GREEN: "c"}), "1 .. 2"),
    (dict(region_prompts={}), "1 .. 2"),
    (dict(region_prompts={RED: "a"}, region_base_ratio=1.5), r"\[0, 1\]"),
    (dict(region_prompts={RED: "a"}, region_base_ratio=-0.1), r"\[0, 1\]"),
    (dict(region_prompts={RED: " ".join(["word"] * 76)}), "75-token"),
])
def test_region_argument_errors(kwargs, match):
    kw = dict(kwargs)
    beta = kw.pop("region_base_ratio", 0.2)
    with pytest.raises(ValueError, match=match):
        _encode(kw.pop("region_prompts"), beta, **kw)


def test_long_base_prompt_and_unaligned_maps_raise():
    s = SETTINGS["cat_dog"]
    with pytest.raises(ValueError, match="75-token"):
        C._encode_text_color_inputs(RandomTextEncoder(32), TOK, "cpu", color_map_image("cat_dog", 128),
                                    dict(s["ctx"]), " ".join(["word"] * 80), "", region_prompts={RED: "a"})
    with pytest.raises(ValueError, match="multiples of 64"):
        C._encode_text_color_inputs(RandomTextEncoder(32), TOK, "cpu", _two_region_map(96, 128), {RED: "x,1"}, "x",
                                    "", region_prompts={RED: "a"})


def test_public_functions_reject_region_prompts_they_cannot_run():
    img = color_map_image("cat_dog", 128)
    with pytest.raises(ValueError, match="attention recording"):
        PL.paint_with_words({RED: "x,1"}, img, "x", region_prompts={RED: "a"}, return_attention_maps=True)
    with pytest.raises(ValueError, match="1 .. 2"):
        PL.paint_with_words({RED: "x,1"}, img, "x", region_prompts={RED: "a", BLUE: "b", GREEN: "c"})
    with pytest.raises(ValueError, match="max_prompt_chunks"):
        PL.paint_with_words_inpaint({RED: "x,1"}, img, img, img, "x", region_prompts={RED: "a"}, max_prompt_chunks=3)
    with pytest.raises(ValueError, match=r"settings\[0\]"):
        PL.paint_with_words_batch([dict(color_map_image=img, region_prompts={RED: "a"}, region_base_ratio=2.0)])


def test_region_entry_points_check_their_arguments():
    L = _native.lib()
    buf = (ctypes.c_char * 4096)()
    p16 = (ctypes.addressof(buf) + 15) // 16 * 16
    common = (p16, p16, p16, p16, 1, 8, 64)
    for fn, stat in ((L.pww_xattn_fused_region_f16, 0), (L.pww_xattn_fused_region_bf16, 0),
                     (L.pww_xattn_fused_region_multi_f16, None), (L.pww_xattn_fused_region_multi_bf16, None)):
        def call(T, w, ws, q=p16):
            return fn(q, *common[1:], T, 40, 20480, 320, T * 320, 320, 20480, 320, None, 0, 0, None, None, stat, None,
                      0.158, None, None, 0, None, w, ws)
        assert call(77, p16, 64 * 3) == -2                        # one chunk: no region mode
        assert call(200, p16, 64 * 3) == -2
        assert call(154, None, 64 * 2) == -1                      # no weights
        assert call(154, p16 + 2, 64 * 2) == -1                   # misaligned weights
        assert call(231, p16, 64 * 3 - 1) == -1                   # stride below N * k
        assert call(154, p16, 64 * 2, q=None) == -1


def test_oracle_identical_chunks_equal_one_softmax_in_fp64():
    g = torch.Generator().manual_seed(3)
    N, H, D = 37, 2, 8
    q = torch.randn(1, N, H * D, generator=g, dtype=torch.float64)
    k1 = torch.randn(1, 77, H * D, generator=g, dtype=torch.float64)
    v1 = torch.randn(1, 77, H * D, generator=g, dtype=torch.float64)
    qh, kh, vh = O._h2b(q, H), O._h2b(k1, H), O._h2b(v1, H)
    ref = O._b2h(torch.matmul((torch.matmul(qh, kh.transpose(-1, -2)) * D ** -0.5).softmax(-1), vh), H)
    for kc in (2, 3):
        w = torch.rand(N, kc, generator=g, dtype=torch.float64)
        w = w / w.sum(1, keepdim=True)
        got = RO.region_attention_core(q, k1.repeat(1, kc, 1), v1.repeat(1, kc, 1), H, D ** -0.5, w,
                                       dtype=torch.float64)
        assert (got - ref).abs().max().item() < 1e-12


def test_oracle_without_weights_is_the_first_chunk_alone():
    g = torch.Generator().manual_seed(4)
    q = torch.randn(1, 10, 16, generator=g)
    k = torch.randn(1, 154, 16, generator=g)
    v = torch.randn(1, 154, 16, generator=g)
    got = RO.region_attention_core(q, k, v, 2, 0.35, None)
    ref = O.attention_core(q, k[:, :77], v[:, :77], 2, 0.35)
    assert torch.allclose(got, ref, atol=1e-6)


def test_batch_groups_keep_region_entries_apart():
    keys = [(8, 8, 154, False), (8, 8, 154, True), (8, 8, 154, True), (8, 8, 231, True)]
    assert PL.batch_groups(keys, 8) == [[0], [1, 2], [3]]
