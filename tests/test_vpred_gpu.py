"""Guidance rescale and v-prediction on the GPU: `pww_sampler_update_rescale` against float64 statistics and against
the same step written as torch fp32 ops, the plain update where phi = 0, batch and position invariance; PwWSampler with
v-prediction schedulers against `reference_rescale_loop`; graphs, launch counts and the public API."""
import functools
import math

import pytest
import torch

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle import rescale_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.pipeline import _BETA, PwWSampler, _dtype_code, ancestral_noise
from paint_with_words_sd_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                                EulerDiscreteScheduler, LMSDiscreteScheduler)
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests.fixtures import SETTINGS, color_map_image, moon_mask_image
from tests.test_samplers_gpu import _WithNoise

pytestmark = pytest.mark.gpu
WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
V = "v_prediction"
SAMPLERS = {"lms": LMSDiscreteScheduler, "euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler,
            "dpmpp_2m": DPMSolverMultistepScheduler,
            "dpmpp_2m_karras": functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=True)}


def _scheduler(name, steps, prediction_type=V):
    sch = SAMPLERS[name](**KW, prediction_type=prediction_type)
    sch.set_timesteps(steps)
    return sch


def _contexts(m):
    g = torch.Generator().manual_seed(0)
    return ([{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)],
            [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)])


# ---- the kernel ------------------------------------------------------------------------------------------------------
def _outputs(m, h, w, dtype, layout, steps, seed):
    """`steps` UNet outputs [2m, 4, h, w] in `dtype` and `layout`, uncond rows scaled apart from cond rows, with a
    per-image offset so |mean| is well above 0."""
    g = torch.Generator().manual_seed(seed)
    outs = []
    for _ in range(steps):
        x = torch.randn(2 * m, 4, h, w, generator=g) + torch.linspace(-2, 3, 2 * m).view(2 * m, 1, 1, 1)
        x[m:] *= 0.6
        x = x.to("cuda", dtype)
        if layout == "channels_last":
            x = x.contiguous(memory_format=torch.channels_last)
        elif layout == "strided":           # channel stride h*w, pixel strides (1, h): the arbitrary-stride path
            x = x.transpose(2, 3).contiguous().transpose(2, 3)
        outs.append(x)
    return outs


class _Run:
    """The sampler state one kernel run needs (step rows, history, noise, guidance, phi) from a PwWSampler over m
    images that is never stepped."""

    def __init__(self, name, m, h, w, phis, steps, seed=0):
        g = torch.Generator().manual_seed(seed + 17)
        conds, unconds = _contexts(m)
        self.lat0 = (torch.randn(m, 4, h, w, generator=g) * 14.6).cuda()
        self.s = PwWSampler(torch.nn.Linear(1, 1).cuda(), _scheduler(name, steps), conds, unconds, self.lat0, WF,
                            [7.5 - 1.5 * i for i in range(m)], use_graph=False, noise_seed=list(range(100, 100 + m)),
                            guidance_rescale=phis)
        self.phi = torch.tensor(phis, dtype=torch.float32, device="cuda")
        self.m, self.h, self.w = m, h, w

    def kernel(self, outs, plain=False):
        """The native run over every step: (latents, per-step stats [steps, m, 3])."""
        s, m, h, w = self.s, self.m, self.h, self.w
        L = _native.lib()
        lat, hist = self.lat0.clone(), torch.zeros_like(s._derivs)
        stats = []
        for i, eps in enumerate(outs):
            p = s._rows[i].clone()
            st = torch.full((m, 3), float("nan"), device="cuda")
            args = (eps.data_ptr(), _dtype_code(eps.dtype), *eps.stride(), lat.data_ptr(), hist.data_ptr(), s._hist_len,
                    None if s._noise is None else s._noise.data_ptr(), s._gscale.data_ptr(), p[_BETA:].data_ptr(),
                    p[s._form:].data_ptr())
            if plain:
                _native.check(L.pww_sampler_update(*args, m, h, w, None), "pww_sampler_update")
            else:
                _native.check(L.pww_sampler_update_rescale(*args, self.phi.data_ptr(), st.data_ptr(), m, h, w, None),
                              "pww_sampler_update_rescale")
            stats.append(st)
        torch.cuda.synchronize()
        return lat, torch.stack(stats)

    def torch_ops(self, outs, ks):
        """The same run as torch fp32 ops in the kernel's order, with the kernel's k of every step."""
        s, m = self.s, self.m
        lat, ring = self.lat0.clone(), torch.zeros_like(s._derivs)
        L = ring.shape[0]
        for i, eps in enumerate(outs):
            r = [float(v) for v in s._rows[i].tolist()]
            alpha, a, b, gamma, slot, nrow = r[-6:]
            beta = r[3:7]
            e = eps.float()
            e = e[m:] + s._gscale * (e[:m] - e[m:])
            k = ks[i].view(m, 1, 1, 1)
            e = torch.where(self.phi.view(m, 1, 1, 1) != 0, k * e, e)
            q = b * e if a == 0 else a * lat + b * e
            ring[int(slot)].copy_(q)
            acc = beta[0] * q
            for j in range(1, L):
                acc = acc + beta[j] * ring[(int(slot) - j) % L]
            out = lat + acc if alpha == 1 else alpha * lat + acc
            if gamma != 0 and s._noise is not None:
                out = out + gamma * s._noise[int(nrow)]
            lat = out
        return lat


def _check_stats(run, outs, stats):
    """std(cond), std(cfg) and k of every image and step within 1e-5 of float64 over the kernel's own fp32 values."""
    m, s = run.m, run.s
    for i, eps in enumerate(outs):
        e = eps.float()
        cfg = e[m:] + s._gscale * (e[:m] - e[m:])
        sc = e[:m].double().flatten(1).std(1)
        sf = cfg.double().flatten(1).std(1)
        phi = run.phi.double()
        k = torch.where(phi != 0, phi * sc / sf + (1 - phi), torch.ones_like(phi))
        want = torch.stack([sc, sf, k], 1)
        rel = ((stats[i].double() - want).abs() / want.abs()).max().item()
        assert rel < 1e-5, (i, rel)


def _kernel_case(name, m, hw, dtype, layout, phis, steps=4):
    h, w = hw
    run = _Run(name, m, h, w, phis, steps, seed=h * 100 + w)
    outs = _outputs(m, h, w, dtype, layout, steps, seed=h * 7 + w)
    lat, stats = run.kernel(outs)
    assert torch.isfinite(lat).all() and torch.isfinite(stats).all()
    _check_stats(run, outs, stats)
    assert torch.equal(lat, run.torch_ops(outs, stats[:, :, 2]))
    # phi = 0 images: exactly the plain update
    plain, _ = run.kernel(outs, plain=True)
    zero = [i for i, p in enumerate(phis) if p == 0]
    assert torch.equal(lat[zero], plain[zero])
    if len(zero) < m:
        assert not torch.equal(lat, plain)
    return run, outs, lat, stats


SIZES = [(8, 8), (33, 47), (64, 64), (96, 96), (128, 128)]


@pytest.mark.parametrize("name", list(SAMPLERS))
@pytest.mark.parametrize("hw", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_rescale_kernel_every_sampler_and_size(name, hw):
    _kernel_case(name, 3, hw, torch.float16, "channels_last", [0.7, 0.0, 1.0])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("layout", ["channels_last", "contiguous", "strided"])
@pytest.mark.parametrize("hw", [(33, 47), (64, 64), (15, 17)], ids=["33x47", "64x64", "15x17"])
def test_rescale_kernel_every_dtype_and_layout(dtype, layout, hw):
    _kernel_case("euler_a", 2, hw, dtype, layout, [0.0, 0.7])


def test_rescale_kernel_with_every_phi_zero_is_the_plain_update():
    _kernel_case("dpmpp_2m_karras", 3, (40, 56), torch.float16, "channels_last", [0.0, 0.0, 0.0])


@pytest.mark.parametrize("hw", [(64, 64), (96, 96), (33, 47)], ids=["64x64", "96x96", "33x47"])
def test_rescale_kernel_is_batch_and_position_invariant(hw):
    """Image i's latents and stats row are the same bits alone, in a batch of 3 or 8 and at any position."""
    h, w = hw
    steps, m = 3, 8
    phis = [0.7, 0.0, 1.0, 0.3, 0.5, 0.9, 0.0, 0.2]
    run = _Run("lms", m, h, w, phis, steps)
    outs = _outputs(m, h, w, torch.float16, "channels_last", steps, seed=5)
    lat, stats = run.kernel(outs)

    def subset(idx):
        sub = _Run("lms", len(idx), h, w, [phis[i] for i in idx], steps)
        sub.lat0 = run.lat0[idx].clone()
        sub.s._gscale = run.s._gscale[idx].contiguous()
        rows = torch.cat([torch.as_tensor(idx), torch.as_tensor(idx) + m]).cuda()
        sub_outs = [o[rows].contiguous(memory_format=torch.channels_last) for o in outs]
        return sub.kernel(sub_outs)
    for idx in ([2], [5], [0], [6, 2, 4], [7, 1, 3]):
        sl, ss = subset(idx)
        assert torch.equal(sl, lat[idx]), idx
        assert torch.equal(ss, stats[:, idx]), idx


# ---- the sampler against the reference loop ------------------------------------------------------------------------
SIZE, STEPS = 128, 4


def _setup(cfg, name, device, seed=0, image="aurora", steps=STEPS):
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim)
    s = SETTINGS[image]
    _, _, cond, uncond = C._encode_text_color_inputs(enc.to(device), tok, device, color_map_image(image, SIZE),
                                                     dict(s["ctx"]), s["prompt"], "")
    sch = _scheduler(name, steps)
    lat = torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=torch.manual_seed(seed)) * sch.init_noise_sigma
    return cond, uncond, sch, lat


def _img2img(sch, seed=3):
    """img2img latents at the schedule's third timestep: a seeded 'init image' latent noised with add_noise."""
    g = torch.Generator().manual_seed(seed)
    init = torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=g)
    ts = sch.timesteps[2:]
    return sch.add_noise(init, torch.randn(init.shape, generator=g), ts[:1]), ts


def _extra(seed=4):
    g = torch.Generator().manual_seed(seed)
    mask = (torch.rand(1, 1, SIZE // 8, SIZE // 8, generator=g) > 0.5).float()
    return torch.cat([mask, torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=g)], 1)


CASES = [(n, phi, "txt2img") for n in SAMPLERS for phi in (0.0, 0.7)] + \
    [("euler", 0.7, "img2img"), ("dpmpp_2m", 0.7, "inpaint")]


def _reference(case):
    name, phi, mode = case
    cfg = UNetConfig.tiny(in_channels=9) if mode == "inpaint" else UNetConfig.tiny()
    unet = build_unet(cfg, seed=0)
    try:
        oracle_loop.patch_with_oracle(unet)
        cond, uncond, sch, lat = _setup(cfg, name, "cpu")
        ts, extra = None, None
        if mode == "img2img":
            lat, ts = _img2img(sch)
        if mode == "inpaint":
            extra = _extra()
        if name == "euler_a":
            sch = _WithNoise(sch, ancestral_noise([0], (1, 4, SIZE // 8, SIZE // 8), STEPS)[:, 0])
        return rescale_loop.reference_rescale_loop(unet, sch, cond, uncond, lat, WF, 7.5, guidance_rescale=phi,
                                                   timesteps=ts, extra_input=extra)
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")


def _native_run(case, use_graph=True):
    name, phi, mode = case
    cfg = UNetConfig.tiny(in_channels=9) if mode == "inpaint" else UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    cond, uncond, sch, lat = _setup(cfg, name, "cuda")
    ts, extra = None, None
    if mode == "img2img":
        lat, ts = _img2img(sch)
    if mode == "inpaint":
        extra = _extra().cuda()
    try:
        P.patch_unet(unet)
        s = PwWSampler(unet, sch, [cond], [uncond], lat.cuda(), WF, 7.5, use_graph=use_graph, noise_seed=0,
                       guidance_rescale=phi, timesteps=ts, extra_input=extra)
        return s.run().float().cpu()
    finally:
        P.unpatch_all()


@pytest.mark.parametrize("case", CASES, ids=[f"{n}-{phi}-{mode}" for n, phi, mode in CASES])
def test_v_sampler_matches_reference_rescale_loop(case):
    ref = _reference(case)
    out = _native_run(case)
    rel_rmse = ((out - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    assert torch.isfinite(out).all() and rel_rmse < 3e-2, rel_rmse


@pytest.mark.parametrize("name", ["lms", "euler_a", "dpmpp_2m_karras"])
def test_graph_and_eager_give_the_same_bits(name):
    case = (name, 0.7, "txt2img")
    assert torch.equal(_native_run(case, use_graph=True), _native_run(case, use_graph=False))


def test_rescale_keeps_the_launches_per_step():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    launches = []
    try:
        P.patch_unet(unet)
        for phi in (0.0, 0.7, [0.0]):
            cond, uncond, sch, lat = _setup(cfg, "dpmpp_2m", "cuda")
            s = PwWSampler(unet, sch, [cond], [uncond], lat.cuda(), WF, 7.5, guidance_rescale=phi)
            s.run(1)
            launches.append((s.native_launches_per_step, s._rescale is not None))
    finally:
        P.unpatch_all()
    assert launches[0][0] == launches[1][0] == launches[2][0] and launches[0][0] > 2
    assert [r for _, r in launches] == [False, True, False]


# ---- the public API ------------------------------------------------------------------------------------------------
def test_sd21_768_v_prediction_with_rescale_is_finite():
    s = SETTINGS["aurora"]
    try:
        lat = P.paint_with_words(color_context=dict(s["ctx"]), color_map_image=color_map_image("aurora", 768),
                                 input_prompt=s["prompt"], num_inference_steps=3, seed=1, device="cuda:0",
                                 weight_function=WF, hf_model_path="synthetic:sd21", prediction_type=V,
                                 guidance_rescale=0.7, scheduler_type=EulerDiscreteScheduler, return_latents=True)
    finally:
        P.unpatch_all()
    assert lat.shape == (1, 4, 96, 96) and torch.isfinite(lat).all()


def test_batch_with_mixed_rescale_matches_solo_calls():
    a, c = SETTINGS["aurora"], SETTINGS["cat_dog"]
    entries = [dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", 128), input_prompt=a["prompt"],
                    seed=0, weight_function=WF, guidance_rescale=0.7),
               dict(color_context=c["ctx"], color_map_image=color_map_image("cat_dog", 128), input_prompt=c["prompt"],
                    seed=1, weight_function=WF, guidance_scale=5.0),
               dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", 128), input_prompt=a["prompt"],
                    seed=2, weight_function=WF, guidance_rescale=1.0)]
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny", scheduler_type=DPMSolverMultistepScheduler,
                             prediction_type=V)
    try:
        got = P.paint_with_words_batch(entries, num_inference_steps=4, device="cuda:0", preloaded_utils=tools,
                                       return_latents=True)
        refs = [P.paint_with_words(**dict(e, color_context=dict(e["color_context"])), num_inference_steps=4,
                                   device="cuda:0", preloaded_utils=tools, return_latents=True) for e in entries]
    finally:
        P.unpatch_all()
    for i, (x, ref) in enumerate(zip(got, refs)):
        d = (x.float() - ref.float()).abs().max().item()
        assert torch.isfinite(x).all() and d <= 2e-2 * ref.abs().max().item(), (i, d)
    assert not torch.allclose(got[0], got[2])


def test_inpaint_pipeline_class_with_v_prediction_and_rescale():
    s = SETTINGS["aurora"]
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny-inpaint", prediction_type=V)
    vae, unet, enc, tok, sch = tools
    try:
        pipe = P.PaintWithWord_StableDiffusionInpaintPipeline(vae, enc, tok, unet, scheduler=sch)
        out = pipe(s["prompt"], image=color_map_image("aurora", 128), mask_image=moon_mask_image(128),
                   color_map_image=color_map_image("aurora", 128), color_context=dict(s["ctx"]), weight_function=WF,
                   num_inference_steps=4, eta=0.5, output_type="latent", guidance_rescale=0.7)
    finally:
        P.unpatch_all()
    assert pipe.scheduler.config["prediction_type"] == V
    assert out.images.shape == (1, 4, 16, 16) and torch.isfinite(out.images).all()
