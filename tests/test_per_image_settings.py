"""Per-image weight functions and guidance scales without a GPU: the sampler's step table, statistic kinds and map
indices, the batch API's argument rules and grouping, and the argument checks of the `_multi` C entry points."""
import ctypes
import math

import pytest
import torch

from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
from paint_with_words_sd_b200.synthetic import IdentityVAE, RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.weight_function import (STAT_MAX, STAT_STD, UnsupportedWeightFunction, g_of_sigma,
                                                      probe_weight_function)
from tests.fixtures import SETTINGS, color_map_image

WF_MAX = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()          # noqa: E731
WF_STD = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.std()          # noqa: E731
WF_STD2 = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma ** 2) * qk.std()    # noqa: E731
WF_ZERO = lambda w, sigma, qk: 0.0                                               # noqa: E731


def _sampler(fns, scales=7.5, m=None):
    """A CPU sampler over m images of random 77-token contexts and a 16x16 map (the UNet is never called)."""
    m = m if m is not None else (1 if callable(fns) else len(fns))
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(5)
    g = torch.Generator().manual_seed(0)
    conds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g), "CROSS_ATTENTION_WEIGHT_256": torch.rand(256, 77),
              "CROSS_ATTENTION_WEIGHT_ORIG": 0} for _ in range(m)]
    unconds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g), "CROSS_ATTENTION_WEIGHT_256": 0,
                "CROSS_ATTENTION_WEIGHT_ORIG": 0} for _ in range(m)]
    return PL.PwWSampler(torch.nn.Linear(1, 1), sch, conds, unconds, torch.zeros(m, 4, 16, 16), fns, scales,
                         use_graph=False), sch


def test_step_table_holds_every_images_g_and_the_probed_kinds():
    fns = [WF_MAX, WF_STD2, WF_ZERO, WF_STD]
    s, sch = _sampler(fns, [7.5, 5.0, 9.0, 3.0])
    table = s._table.cpu()
    assert table.shape == (len(s.timesteps), 7 + 4)
    for row, t in enumerate(s.timesteps):
        sigma = sch.sigmas[sch.step_index_of(t)]
        for i, f in enumerate(fns):
            want = torch.tensor(g_of_sigma(f, probe_weight_function(f), sigma), dtype=torch.float32)
            assert table[row, 7 + i] == want, (row, i)
    assert table[:, 9].eq(0).all()                                        # the zero function
    assert s._ctx["STAT_KIND"].tolist() == [STAT_MAX, STAT_STD, STAT_MAX, STAT_STD] + [STAT_MAX] * 4
    assert s._ctx["WMAP_INDEX"].tolist() == [0, 1, -1, 3] + [-1] * 4
    assert s._gscale.flatten().tolist() == [7.5, 5.0, 9.0, 3.0]
    # a step copies its row; G_SIGMA holds one value per image of the UNet batch, the uncond ones stay 0
    s._set_step_scalars(2, sch.step_index_of(s.timesteps[2]))
    assert s._ctx["G_SIGMA"].numel() == 8
    assert torch.equal(s._ctx["G_SIGMA"][:4], table[2, 7:]) and s._ctx["G_SIGMA"][4:].eq(0).all()
    assert torch.equal(s._params[:7], table[2, :7])


def test_one_callable_is_the_uniform_case():
    s, _ = _sampler(WF_STD, 6.0, m=3)
    table = s._table
    assert table.shape[1] == 7 + 3
    assert torch.equal(table[:, 7], table[:, 8]) and torch.equal(table[:, 7], table[:, 9])
    assert s._ctx["STAT_KIND"].tolist()[:3] == [STAT_STD] * 3
    assert s._ctx["WMAP_INDEX"].tolist() == [0, 1, 2, -1, -1, -1]
    assert s._gscale.flatten().tolist() == [6.0] * 3 and s.guidance_scale == 6.0
    z, _ = _sampler(WF_ZERO)
    assert z._ctx["WMAP_INDEX"].tolist() == [-1, -1] and z._table[:, 7].eq(0).all()


def test_unsupported_weight_function_names_the_image():
    mixed = lambda w, sigma, qk: w * (qk.max() + qk.std())     # noqa: E731
    with pytest.raises(UnsupportedWeightFunction, match="image 2"):
        _sampler([WF_MAX, WF_STD, mixed])
    with pytest.raises(UnsupportedWeightFunction):
        _sampler(mixed)


def test_per_image_settings_need_one_value_per_image():
    with pytest.raises(ValueError, match="weight_function"):
        _sampler([WF_MAX, WF_STD], m=3)
    with pytest.raises(ValueError, match="guidance_scale"):
        _sampler([WF_MAX, WF_STD], [7.5, 5.0, 3.0])


def test_batch_rejects_unknown_keys_and_img2img():
    base = dict(color_context=dict(SETTINGS["aurora"]["ctx"]), color_map_image=color_map_image("aurora", 64))
    with pytest.raises(ValueError, match="unknown keys"):
        PL.paint_with_words_batch([base, dict(base, guidance=3.0)], preloaded_utils=())
    for key, val in (("init_image", color_map_image("aurora", 64)), ("strength", 0.3)):
        with pytest.raises(ValueError, match="init_image"):
            PL.paint_with_words_batch([dict(base, **{key: val})], preloaded_utils=())
    with pytest.raises(ValueError, match="color_map_image"):
        PL.paint_with_words_batch([{"input_prompt": "a cat"}], preloaded_utils=())


def test_batch_settings_take_paint_with_words_defaults():
    full = PL._batch_settings([{"color_map_image": color_map_image("aurora", 64), "seed": 4}])[0]
    assert set(full) == set(PL.BATCH_SETTING_KEYS)
    assert full["weight_function"] is PL.default_weight_function and full["guidance_scale"] == 7.5
    assert full["seed"] == 4 and full["max_prompt_chunks"] == 1 and full["input_prompt"] == ""


def test_batch_groups_keep_order_and_cap_the_batch():
    keys = ["a", "b", "a", None, "a", "b", "a", None]
    assert PL.batch_groups(keys, 8) == [[0, 2, 4, 6], [1, 5], [3], [7]]
    assert PL.batch_groups(keys, 3) == [[0, 2, 4], [6], [1, 5], [3], [7]]
    assert PL.batch_groups(keys, 1) == [[i] for i in (0, 2, 4, 6, 1, 5, 3, 7)]
    with pytest.raises(ValueError):
        PL.batch_groups(keys, 0)


class _RecordingSampler:
    """Stands in for PwWSampler: records what each sampler gets and returns its latents unchanged."""
    runs = []

    def __init__(self, unet, scheduler, conds, unconds, latents, weight_function, guidance_scale, **kw):
        self.latents = latents
        _RecordingSampler.runs.append(dict(m=len(conds), shape=tuple(latents.shape[-2:]),
                                           T={int(c["CONTEXT_TENSOR"].shape[1]) for c in conds + unconds},
                                           fns=list(weight_function), scales=list(guidance_scale)))

    def run(self):
        return self.latents


def test_batch_groups_entries_by_size_and_text_length(monkeypatch):
    monkeypatch.setattr(PL, "PwWSampler", _RecordingSampler)
    _RecordingSampler.runs = []
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")

    class _UNet:
        in_channels = 4
    tools = (IdentityVAE(), _UNet(), RandomTextEncoder(32), SimpleWordTokenizer(), sch)
    long_prompt = " ".join(["word"] * 90) + " aurora"
    a, c = SETTINGS["aurora"], SETTINGS["cat_dog"]
    entries = [
        dict(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 64), input_prompt=a["prompt"],
             seed=0, weight_function=WF_MAX),
        dict(color_context=dict(c["ctx"]), color_map_image=color_map_image("cat_dog", 128), input_prompt=c["prompt"],
             seed=1, weight_function=WF_STD2, guidance_scale=5.0),
        dict(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 64), input_prompt=long_prompt,
             seed=2, max_prompt_chunks=2),
        dict(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 64), input_prompt=a["prompt"],
             seed=3, weight_function=WF_ZERO, guidance_scale=9.0),
        dict(color_context=dict(c["ctx"]), color_map_image=color_map_image("cat_dog", 128), input_prompt=c["prompt"],
             seed=4),
    ]
    before = [dict(e["color_context"]) for e in entries]
    out = PL.paint_with_words_batch(entries, num_inference_steps=3, device="cpu", preloaded_utils=tools,
                                    max_batch_size=8, return_latents=True)
    runs = _RecordingSampler.runs
    assert [(r["m"], r["shape"], r["T"]) for r in runs] == [(2, (8, 8), {77}), (2, (16, 16), {77}), (1, (8, 8), {154})]
    assert runs[0]["fns"] == [WF_MAX, WF_ZERO] and runs[0]["scales"] == [7.5, 9.0]
    assert runs[1]["fns"] == [WF_STD2, PL.default_weight_function] and runs[1]["scales"] == [5.0, 7.5]
    # input order, each image its own seeded noise; the caller's colour contexts are not mutated
    assert [tuple(o.shape) for o in out] == [(1, 4, 8, 8), (1, 4, 16, 16), (1, 4, 8, 8), (1, 4, 8, 8), (1, 4, 16, 16)]
    for i, e in enumerate(entries):
        h = e["color_map_image"].size[1] // 8
        noise = torch.randn((1, 4, h, h), generator=torch.manual_seed(e["seed"])) * sch.init_noise_sigma
        assert torch.equal(out[i], noise), i
        assert e["color_context"] == before[i]
    _RecordingSampler.runs = []
    PL.paint_with_words_batch(entries, num_inference_steps=3, device="cpu", preloaded_utils=tools, max_batch_size=1,
                              return_latents=True)
    assert [r["m"] for r in _RecordingSampler.runs] == [1] * 5


def _buf():
    buf = (ctypes.c_char * 8192)()
    return buf, (ctypes.addressof(buf) + 15) // 16 * 16


def test_multi_entry_points_validate_without_a_gpu():
    L = _native.lib()
    assert L.pww_version() == 300
    buf, p = _buf()
    B, H, N, T, D = 2, 8, 64, 77, 40
    C = H * D
    big_ws = L.pww_xattn_fused_workspace_bytes()
    # fused: a map with a null kind or G array is a bad argument; with both, the (too small) workspace is what fails
    fused = lambda T_, kinds, g, ws: L.pww_xattn_fused_multi_f16(   # noqa: E731
        p, p, p, p, B, H, N, T_, D, N * C, C, T_ * C, C, N * C, C, p, N * 32, 1, p, p, kinds, g, 0.158, p, p, ws, None)
    assert fused(T, None, p, big_ws) == -1
    assert fused(T, p, None, big_ws) == -1
    assert fused(T, p, p, 16) == -4
    assert fused(81, p, p, big_ws) == -2
    # no map: plain attention, the arrays are not needed (T = 81 is still unsupported)
    assert L.pww_xattn_fused_multi_f16(p, p, p, p, B, H, N, 81, D, N * C, C, 81 * C, C, N * C, C, None, 0, 0, None,
                                       None, None, None, 0.158, None, None, 0, None) == -2
    # stats: the kind array is always needed
    stats = lambda T_, kinds, ws: L.pww_xattn_stats_multi_f16(   # noqa: E731
        p, p, B, H, N, T_, D, N * C, C, T_ * C, C, kinds, None, p, p, ws, None)
    assert stats(T, None, 1 << 30) == -1
    assert stats(T, p, 16) == -4
    assert stats(81, p, 1 << 30) == -2
    # forward: a map with a null G array
    fwd = lambda T_, g: L.pww_xattn_fwd_multi_f16(   # noqa: E731
        p, p, p, p, B, H, N, T_, D, N * C, C, T_ * C, C, N * C, C, p, N * T_, p, p, g, 0.158, None)
    assert fwd(T, None) == -1
    assert fwd(81, p) == -2
