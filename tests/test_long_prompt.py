"""Long prompts without a GPU: chunked tokenization (2 / 3 CLIP windows of 77 tokens), the maps built on the chunked ids
against the unmodified reference (tests/golden/long_prompt.npz), the chunked packed-map layout and the ABI's key-length
validation."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import pww_oracle as O
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import CrossAttention
from tests.fixtures import GOLDEN, SETTINGS, color_map_image, exact_digest
from tests.golden.make_long_prompt_golden import LONG_AURORA_PROMPT

TOK = SimpleWordTokenizer()
BOS, EOS = TOK.bos_token_id, TOK.eos_token_id


@pytest.fixture(scope="module")
def long_golden():
    return np.load(os.path.join(GOLDEN, "long_prompt.npz"))


def _encode(prompt, chunks, ctx=None, size=128):
    s = SETTINGS["aurora"]
    return C._encode_text_color_inputs(RandomTextEncoder(64), TOK, "cpu", color_map_image("aurora", size),
                                       dict(s["ctx"] if ctx is None else ctx), prompt, "", max_prompt_chunks=chunks)


def _labels(ctx):
    return [v.rpartition(",")[0] for v in ctx.values()]


def _words(n):
    return " ".join(f"w{i}" for i in range(n))


def test_short_prompt_gives_identical_dicts_for_every_chunk_limit():
    prompt = SETTINGS["aurora"]["prompt"]
    assert len(TOK(prompt)["input_ids"]) - 2 <= 75
    one = _encode(prompt, 1)
    for chunks in (2, 3):
        other = _encode(prompt, chunks)
        assert one[0] == other[0]
        for a, b in zip(one[2:], other[2:]):
            assert a.keys() == b.keys()
            for k in a:
                if isinstance(a[k], torch.Tensor):
                    assert torch.equal(a[k], b[k]), k
                else:
                    assert a[k] == b[k], k


def test_long_prompt_fills_two_chunks():
    assert 75 < len(TOK(LONG_AURORA_PROMPT)["input_ids"]) - 2 <= 150
    ids = C.chunk_prompt(TOK, LONG_AURORA_PROMPT, _labels(SETTINGS["aurora"]["ctx"]), 3)[0]
    assert ids.shape == (154,)
    for c in range(2):
        chunk = ids[77 * c:77 * (c + 1)].tolist()
        assert chunk[0] == BOS and EOS in chunk[1:]
        end = chunk.index(EOS, 1)
        assert all(t == EOS for t in chunk[end:])                 # padded the way the tokenizer pads one window
    _, _, cond, uncond = _encode(LONG_AURORA_PROMPT, 3)
    enc = RandomTextEncoder(64)
    assert cond["CONTEXT_TENSOR"].shape == (1, 154, 64) and uncond["CONTEXT_TENSOR"].shape == (1, 154, 64)
    # every chunk is encoded on its own
    assert torch.equal(cond["CONTEXT_TENSOR"][:, 77:], enc(ids[None, 77:])[0])
    empty = torch.tensor([[BOS, EOS] + [EOS] * 75])
    assert torch.equal(uncond["CONTEXT_TENSOR"][:, 77:], enc(empty)[0])
    for key, w in cond.items():
        if key.startswith("CROSS_ATTENTION_WEIGHT_") and key != "CROSS_ATTENTION_WEIGHT_ORIG":
            assert w.shape[-1] == 154
    assert cond["CROSS_ATTENTION_WEIGHT_ORIG"].shape[-1] == 154


def test_no_label_straddles_a_chunk_boundary():
    # "full moon" sits at prompt tokens 74-75: a plain 75-token cut would split it
    ids_flat = TOK(LONG_AURORA_PROMPT)["input_ids"][1:-1]
    moon = TOK("full moon")["input_ids"][1:-1]
    assert ids_flat[74:76] == moon
    ids = C.chunk_prompt(TOK, LONG_AURORA_PROMPT, _labels(SETTINGS["aurora"]["ctx"]), 3)[0].tolist()
    for label in _labels(SETTINGS["aurora"]["ctx"]):
        lab = TOK(label)["input_ids"][1:-1]
        assert len(C._match_positions(ids, lab)) == len(C._match_positions(ids_flat, lab)), label
    assert ids[77:80] == [BOS] + moon                              # the first window ended before the label
    # the window rule on its own, with overlapping spans
    win = C._prompt_windows(list(range(200)), [[70, 71, 72, 73, 74, 75, 76], [74, 75, 76, 77, 78]], 3, 75)
    assert [len(w) for w in win] == [70, 75, 55] and sum(win, []) == list(range(200))


def test_label_longer_than_a_window_raises():
    ctx = {(7, 9, 182): _words(80) + ",0.5"}
    with pytest.raises(ValueError):
        C.chunk_prompt(TOK, _words(120), _labels(ctx), 2)
    with pytest.raises(ValueError):
        _encode(_words(120), 2, ctx=ctx)
    with pytest.raises(ValueError):
        _encode(_words(20), 4)


def test_truncation_past_three_chunks():
    ids = C.chunk_prompt(TOK, _words(300), [], 3)[0].tolist()
    assert len(ids) == 231
    flat = TOK(_words(300))["input_ids"][1:-1]
    body = [t for t in ids if t not in (BOS, EOS)]
    assert body == flat[:225]
    assert C.chunk_prompt(TOK, _words(300), [], 2).shape == (1, 154)


def test_long_prompt_maps_match_reference(long_golden):
    g = long_golden
    s = SETTINGS["aurora"]
    ids = C.chunk_prompt(TOK, LONG_AURORA_PROMPT, _labels(s["ctx"]), 3)
    assert ids[0].tolist() == g["ids"].tolist()
    sep, _, _ = C._image_context_seperator(color_map_image("aurora", 512), dict(s["ctx"]), TOK)
    text_input = {"input_ids": ids}
    for r in (8, 16, 32, 64):
        got = C._tokens_img_attention_weight(sep, text_input, ratio=r)
        assert torch.equal(got, torch.from_numpy(g[f"w{r}"])), f"ratio {r} not bit-exact"
    orig = C._tokens_img_attention_weight(sep, text_input, ratio=1, original_shape=True)
    assert list(orig.shape) == g["orig_shape"].tolist()
    assert np.array_equal(exact_digest(orig), g["orig_digest"])


@torch.no_grad()
def test_oracle_inj_forward_at_154_keys_matches_reference(long_golden):
    g = long_golden
    heads = int(g["heads"])
    Cd, dc = g["x"].shape[-1], g["ctx"].shape[-1]
    attn = CrossAttention(Cd, dc, heads, Cd // heads)
    for name, p in attn.named_parameters():
        p.data = torch.from_numpy(g[f"attn.{name}"])
    x, ctx, w = (torch.from_numpy(g[k]) for k in ("x", "ctx", "w"))
    sigma = torch.tensor(float(g["sigma"]))
    fns = {"max": lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max(),
           "std": lambda w, sigma, qk: 0.5 * w * math.log(1 + sigma) * qk.std()}
    for name, f in fns.items():
        c = {"CONTEXT_TENSOR": ctx, f"CROSS_ATTENTION_WEIGHT_{x.shape[1]}": w, "CROSS_ATTENTION_WEIGHT_ORIG": 0,
             "SIGMA": sigma, "WEIGHT_FUNCTION": f}
        assert torch.allclose(O.inj_forward(attn, x, c), torch.from_numpy(g[f"out_dict_{name}"]), atol=2e-6, rtol=1e-5)


@pytest.mark.parametrize("T", [154, 231])
def test_pack_round_trip_chunked_layout(T):
    """Bit-exact on maps whose values hi + lo represents exactly (the reference maps round-trip to 2^-21, see
    test_host_logic)."""
    gen = torch.Generator().manual_seed(T)
    N = 333
    w = torch.zeros(2, N, T)
    for b in range(2):
        for r in range(6):
            col = torch.round(torch.rand(N, generator=gen) * 3 * 1024) / 1024     # exact in fp16 hi + lo
            for t in torch.randperm(T, generator=gen)[:4]:
                w[b, :, t] += col
    packed = C.pack_weight_map(w)
    assert packed is not None
    mpack, cidx = packed
    k = T // 77
    assert cidx.shape == (2, 80 * k)
    for c in range(k):
        assert (cidx[:, 80 * c + 77:80 * c + 80] == -1).all()
    assert torch.equal(C.unpack_weight_map(mpack, cidx, T), w)
    # token 77 c + j at column 80 c + j
    nz = (w[0] != 0).any(0).nonzero().flatten()
    assert ((cidx[0, nz // 77 * 80 + nz % 77]) >= 0).all()
    for bad in (81, 128, 155, 200):
        assert C.pack_weight_map(torch.zeros(1, 4, bad)) is None


def test_pack_short_maps_unchanged():
    gen = torch.Generator().manual_seed(3)
    w = torch.zeros(1, 64, 77)
    w[0, :, 5:8] = torch.round(torch.rand(64, 1, generator=gen) * 1024) / 1024
    mpack, cidx = C.pack_weight_map(w)
    assert cidx.shape == (1, 80) and (cidx[0, 77:] == -1).all() and (cidx[0, 5:8] == 0).all()
    assert torch.equal(C.unpack_weight_map(mpack, cidx, 77), w)


def test_orig_fallback_is_generic_in_tokens():
    gen = torch.Generator().manual_seed(1)
    w_orig = torch.rand(24, 24, 154, generator=gen)
    full = C.expand_orig_weight_map(w_orig, 64)
    assert full.shape == (64, 154)
    # columns are interpolated independently (to the last ulp: the CPU kernels vectorise over channels)
    assert torch.allclose(full[:, :77], C.expand_orig_weight_map(w_orig[..., :77].contiguous(), 64), atol=1e-6, rtol=0)
    assert torch.equal(full, O.orig_map_fallback(w_orig, 64))


@pytest.mark.parametrize("T", [155, 160, 232, 308])
def test_abi_rejects_other_long_key_counts(T):
    L = _native.lib()
    buf = (ctypes.c_char * 4096)()
    p16 = (ctypes.addressof(buf) + 15) // 16 * 16
    assert L.pww_xattn_fwd_f16(p16, p16, p16, p16, 1, 8, 64, T, 40, 20480, 320, 320 * T, 320, 20480, 320,
                               None, 0, None, None, None, 0.158, None) == -2
    assert L.pww_xattn_stats_f16(p16, p16, 1, 8, 64, T, 40, 20480, 320, 320 * T, 320, 0, None, p16, p16, 1 << 20,
                                 None) == -2
    assert L.pww_xattn_fused_f16(p16, p16, p16, p16, 1, 8, 64, T, 40, 20480, 320, 320 * T, 320, 20480, 320,
                                 None, 0, 0, None, None, 0, None, 0.158, None, None, 0, None) == -2


def test_workspace_sizes_do_not_depend_on_tokens():
    L = _native.lib()
    assert L.pww_xattn_workspace_bytes(2, 8, 4096, 77, 40) == L.pww_xattn_workspace_bytes(2, 8, 4096, 231, 40)
    assert L.pww_version() >= 200
