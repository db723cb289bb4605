"""The native sampler step on the GPU: `pww_sampler_input` + `pww_sampler_update` against the previous torch step tail
(LMS, bitwise) and against a torch restatement of the step form (Euler, Euler ancestral, DPM++ 2M, bitwise), the
samplers against the reference loop, a point-mass UNet, batching, the public API and the launch count."""
import functools
import math

import pytest
import torch

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.pipeline import PwWSampler, ancestral_noise
from paint_with_words_sd_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                                EulerDiscreteScheduler, LMSDiscreteScheduler)
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests.fixtures import SETTINGS, color_map_image, moon_mask_image

pytestmark = pytest.mark.gpu
WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
DPM_KARRAS = functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=True)
SAMPLERS = {"lms": LMSDiscreteScheduler, "euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler,
            "dpmpp_2m": DPMSolverMultistepScheduler, "dpmpp_2m_karras": DPM_KARRAS}


class _Out:
    def __init__(self, sample):
        self.sample = sample


class ReplayUNet(torch.nn.Module):
    """Returns the next of a list of precomputed eps tensors and records every input it is given."""

    def __init__(self, eps, dtype):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, dtype=dtype, device="cuda"))
        self.eps, self.inputs = eps, []

    def forward(self, x, t, encoder_hidden_states=None):
        self.inputs.append(x.clone())
        return _Out(self.eps[len(self.inputs) - 1])


def _contexts(m):
    g = torch.Generator().manual_seed(0)
    return ([{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)],
            [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)])


def _scheduler(cls, steps):
    sch = cls(**KW)
    sch.set_timesteps(steps)
    return sch


def _old_lms_tail(lat, derivs, params, gscale, eps, extra, dtype, m):
    """The previous release's step around the UNet, expression by expression: returns the UNet input it built and
    updates lat / derivs in place."""
    x = lat * params[1]
    if extra is not None:
        x = torch.cat([x, extra], dim=1)
    x2 = torch.cat([x, x], 0).to(dtype)
    e = eps.float()
    eps_c, eps_u = e[:m], e[m:]
    noise_pred = eps_u + gscale * (eps_c - eps_u)
    derivs.copy_(torch.roll(derivs, 1, 0))
    derivs[0].copy_(noise_pred)
    upd = (params[3:7].view(4, 1, 1, 1, 1) * derivs).sum(0)
    lat.add_(upd)
    return x2


def _step_form_tail(lat, ring, row, gscale, eps, extra, dtype, m, i, noise):
    """The step form as separate torch ops in the kernel's order (row: one uploaded step row)."""
    r = [float(v) for v in row.tolist()]
    alpha, a, b, gamma, slot, nrow = r[-6:]
    beta, L = r[3:7], ring.shape[0]
    x = lat * row[1]
    if extra is not None:
        x = torch.cat([x, extra], dim=1)
    x2 = torch.cat([x, x], 0).to(dtype)
    e = eps.float()
    g = gscale.view(m, 1, 1, 1)
    e = e[m:] + g * (e[:m] - e[m:])
    q = b * e if a == 0 else a * lat + b * e
    ring[int(slot)].copy_(q)
    s = beta[0] * q
    for k in range(1, L):
        s = s + beta[k] * ring[(int(slot) - k) % L]
    out = lat + s if alpha == 1 else alpha * lat + s
    if gamma != 0 and noise is not None:
        out = out + gamma * noise[int(nrow)]
    lat.copy_(out)
    return x2


SIZES = [(16, 16), (64, 64), (96, 96), (40, 56), (15, 17)]     # 15x17: h*w % 4 != 0, one pixel per thread


@pytest.mark.parametrize("sampler", ["lms", "euler", "euler_a", "dpmpp_2m_karras"])
@pytest.mark.parametrize("m", [1, 3, 8])
@pytest.mark.parametrize("hw", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
@pytest.mark.parametrize("inpaint", [False, True], ids=["txt2img", "inpaint"])
@pytest.mark.parametrize("layout", ["channels_last", "contiguous"])
def test_native_step_is_bitwise_equal_to_torch(sampler, m, hw, inpaint, layout):
    _bitwise_case(sampler, m, hw, inpaint, layout, torch.float16, steps=30)


@pytest.mark.parametrize("sampler", ["lms", "euler_a", "dpmpp_2m"])
@pytest.mark.parametrize("layout", ["channels_last", "contiguous"])
def test_native_step_is_bitwise_equal_to_torch_fp32_unet(sampler, layout):
    _bitwise_case(sampler, 3, (40, 56), True, layout, torch.float32, steps=12)


def _bitwise_case(sampler, m, hw, inpaint, layout, dtype, steps):
    h, w = hw
    g = torch.Generator().manual_seed(m * 1000 + h * 10 + w)
    fmt = torch.channels_last if layout == "channels_last" else torch.contiguous_format
    eps = [(torch.randn(2 * m, 4, h, w, generator=g)).to("cuda", dtype).contiguous(memory_format=fmt)
           for _ in range(steps)]
    lat0 = torch.randn(m, 4, h, w, generator=g) * 14.6
    extra = torch.randn(m, 5, h, w, generator=g).cuda() if inpaint else None
    sch = _scheduler(SAMPLERS[sampler], steps)
    conds, unconds = _contexts(m)
    unet = ReplayUNet(eps, dtype)
    scales = [7.5 - 1.5 * i for i in range(m)]
    s = PwWSampler(unet, sch, conds, unconds, lat0.cuda(), WF, scales, extra_input=extra, use_graph=False,
                   noise_seed=list(range(m)))
    lat = lat0.cuda()
    hist = torch.zeros_like(s._derivs)
    with torch.no_grad():
        for i in range(steps):
            s.step()
            row = s._rows[i]
            if sampler == "lms":
                params = row[:7]
                x2 = _old_lms_tail(lat, hist, params, s._gscale, eps[i], extra, dtype, m)
            else:
                x2 = _step_form_tail(lat, hist, row, s._gscale, eps[i], extra, dtype, m, i, s._noise)
            assert torch.equal(unet.inputs[i], x2), f"UNet input differs at step {i}"
            assert torch.equal(s.latents, lat), f"latents differ at step {i}"
    assert torch.isfinite(lat).all()


# ---- against the reference loop -------------------------------------------------------------------------------------
SIZE, STEPS = 128, 4


def _setup(cfg, cls, device, seed=0, name="aurora"):
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim)
    s = SETTINGS[name]
    _, _, cond, uncond = C._encode_text_color_inputs(enc.to(device), tok, device, color_map_image(name, SIZE),
                                                     dict(s["ctx"]), s["prompt"], "")
    sch = _scheduler(cls, STEPS)
    lat = torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=torch.manual_seed(seed)) * sch.init_noise_sigma
    return cond, uncond, sch, lat


class _WithNoise:
    """The scheduler with `noise=` passed to every `step`, as the sampler draws it (draws 1..n of the seed)."""

    def __init__(self, sch, noise):
        self._sch, self._noise, self._k = sch, noise, 0

    def __getattr__(self, name):
        return getattr(self._sch, name)

    def step(self, eps, t, x):
        out = self._sch.step(eps, t, x, noise=self._noise[self._k])
        self._k += 1
        return out


@pytest.fixture(scope="module")
def reference_loops():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0)
    refs = {}
    try:
        oracle_loop.patch_with_oracle(unet)
        for name in ("euler", "euler_a", "dpmpp_2m", "dpmpp_2m_karras"):
            cond, uncond, sch, lat = _setup(cfg, SAMPLERS[name], "cpu")
            if name == "euler_a":
                sch = _WithNoise(sch, ancestral_noise([0], (1, 4, SIZE // 8, SIZE // 8), STEPS)[:, 0])
            refs[name] = oracle_loop.reference_denoise_loop(unet, sch, cond, uncond, lat, WF)
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")
    return refs


@pytest.mark.parametrize("name", ["euler", "euler_a", "dpmpp_2m", "dpmpp_2m_karras"])
@pytest.mark.parametrize("use_graph", [False, True])
def test_sampler_matches_reference_loop(name, use_graph, reference_loops):
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    cond, uncond, sch, lat = _setup(cfg, SAMPLERS[name], "cuda")
    try:
        P.patch_unet(unet)
        out = PwWSampler(unet, sch, [cond], [uncond], lat.cuda(), WF, 7.5, use_graph=use_graph, noise_seed=0).run()
    finally:
        P.unpatch_all()
    out, ref = out.float().cpu(), reference_loops[name]
    rel_rmse = ((out - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    assert torch.isfinite(out).all() and rel_rmse < 3e-2, rel_rmse


# ---- point mass ------------------------------------------------------------------------------------------------------
class PointMassUNet(torch.nn.Module):
    """eps of a point mass at x0: (x - x0) / sigma, with x recovered from the scaled input; the same for cond and
    uncond, so CFG returns it unchanged."""

    def __init__(self, x0, params):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, device="cuda"))
        self.x0, self.params = x0, params

    def forward(self, x, t, encoder_hidden_states=None):
        lat = x[:, :4] / self.params[1]
        return _Out((lat - torch.cat([self.x0, self.x0])) / self.params[0])


@pytest.mark.parametrize("name", list(SAMPLERS))
@pytest.mark.parametrize("use_graph", [False, True])
def test_point_mass_ends_at_x0(name, use_graph):
    m, steps = 2, 20
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(m, 4, 16, 16, generator=g).cuda()
    sch = _scheduler(SAMPLERS[name], steps)
    lat = x0 + float(sch.sigmas[0]) * torch.randn(m, 4, 16, 16, generator=g).cuda()
    conds, unconds = _contexts(m)
    s = PwWSampler(torch.nn.Linear(1, 1).cuda(), sch, conds, unconds, lat, WF, [7.5, 3.0], use_graph=use_graph,
                   noise_seed=[4, 5])
    s.unet = PointMassUNet(x0, s._params)          # fp32, like the Linear the sampler was built with
    # the last step lands on x0 whatever came before; the deterministic samplers must also stay on the exact trajectory
    # x_i = x0 + sigma_i (x_T - x0) / sigma_T at every step
    with torch.no_grad():
        for i in range(steps):
            s.step()
            if name != "euler_a":
                exact = x0 + float(sch.sigmas[i + 1]) / float(sch.sigmas[0]) * (lat - x0)
                d = (s.latents - exact).abs().max().item()
                assert d < 1e-4 * lat.abs().max().item(), (i, d)
    err = (s.latents - x0).abs().max().item()
    assert err < 1e-4 * x0.abs().max().item() + 1e-5, err


@pytest.mark.parametrize("name", ["lms", "dpmpp_2m_karras"])
def test_channels_last_latents_give_the_same_run(name):
    """The sampler copies latents (and extra_input) to contiguous fp32: a channels-last input gives the same latents."""
    m, h, w, steps = 2, 24, 40, 6
    g = torch.Generator().manual_seed(7)
    eps = [torch.randn(2 * m, 4, h, w, generator=g).to("cuda", torch.float16) for _ in range(steps)]
    lat = (torch.randn(m, 4, h, w, generator=g) * 14.6).cuda()
    extra = torch.randn(m, 5, h, w, generator=g).cuda()
    outs = []
    for fmt in (torch.contiguous_format, torch.channels_last):
        conds, unconds = _contexts(m)
        s = PwWSampler(ReplayUNet(eps, torch.float16), _scheduler(SAMPLERS[name], steps), conds, unconds,
                       lat.contiguous(memory_format=fmt), WF, 7.5, extra_input=extra.contiguous(memory_format=fmt),
                       use_graph=False)
        outs.append(s.run().clone())
    assert torch.equal(outs[0], outs[1]) and torch.isfinite(outs[0]).all()


# ---- batching and the public API -------------------------------------------------------------------------------------
def test_euler_ancestral_batch_equals_solo_runs():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    try:
        P.patch_unet(unet)
        imgs = [_setup(cfg, EulerAncestralDiscreteScheduler, "cuda", seed=i, name=n)
                for i, n in enumerate(("aurora", "cat_dog"))]
        sch = imgs[0][2]
        both = PwWSampler(unet, sch, [x[0] for x in imgs], [x[1] for x in imgs],
                          torch.cat([x[3] for x in imgs]).cuda(), WF, 7.5, noise_seed=[10, 11]).run().clone()
        solo = [PwWSampler(unet, x[2], [x[0]], [x[1]], x[3].cuda(), WF, 7.5, noise_seed=10 + i).run().clone()
                for i, x in enumerate(imgs)]
    finally:
        P.unpatch_all()
    for i in range(2):
        d = (both[i] - solo[i][0]).abs().max().item()
        assert d <= 2e-2 * solo[i].abs().max().item(), (i, d)
    assert not torch.allclose(both[0], both[1])


def test_public_api_runs_every_scheduler_type():
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    s = SETTINGS["aurora"]
    outs = {}
    try:
        for name in SAMPLERS:
            vae, unet, enc, tok, _ = tools
            sch = SAMPLERS[name](**KW)
            outs[name] = P.paint_with_words(color_context=dict(s["ctx"]), color_map_image=color_map_image("aurora", 128),
                                            input_prompt=s["prompt"], num_inference_steps=4, seed=2, device="cuda:0",
                                            weight_function=WF, preloaded_utils=(vae, unet, enc, tok, sch),
                                            return_latents=True)
        img = P.paint_with_words(color_context=dict(s["ctx"]), color_map_image=color_map_image("aurora", 128),
                                 input_prompt=s["prompt"], num_inference_steps=2, device="cuda:0", weight_function=WF,
                                 scheduler_type=DPM_KARRAS, hf_model_path="synthetic:tiny")
    finally:
        P.unpatch_all()
    for name, x in outs.items():
        assert x.shape == (1, 4, 16, 16) and torch.isfinite(x).all(), name
    assert not torch.allclose(outs["euler"], outs["euler_a"]) and not torch.allclose(outs["lms"], outs["dpmpp_2m"])
    assert img.size == (128, 128)


def test_inpaint_with_dpmpp_2m():
    s = SETTINGS["aurora"]
    try:
        lat = P.paint_with_words_inpaint(color_context=dict(s["ctx"]), color_map_image=color_map_image("aurora", 128),
                                         mask_image=moon_mask_image(128), init_image=color_map_image("aurora", 128),
                                         input_prompt=s["prompt"], num_inference_steps=6, strength=0.5,
                                         scheduler_type=DPMSolverMultistepScheduler, weight_function=WF,
                                         hf_model_path="synthetic:tiny-inpaint", return_latents=True)
    finally:
        P.unpatch_all()
    assert lat.shape == (1, 4, 16, 16) and torch.isfinite(lat).all()


def test_batch_api_with_euler_ancestral_matches_solo_calls():
    a, c = SETTINGS["aurora"], SETTINGS["cat_dog"]
    entries = [dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", 128), input_prompt=a["prompt"],
                    seed=0, weight_function=WF),
               dict(color_context=c["ctx"], color_map_image=color_map_image("cat_dog", 128), input_prompt=c["prompt"],
                    seed=1, weight_function=WF, guidance_scale=5.0)]
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny", scheduler_type=EulerAncestralDiscreteScheduler)
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


# ---- launches ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lms", "dpmpp_2m_karras"])
def test_step_is_the_unet_plus_two_native_launches(name):
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    try:
        P.patch_unet(unet)
        cond, uncond, sch, lat = _setup(cfg, SAMPLERS[name], "cuda")
        s = PwWSampler(unet, sch, [cond], [uncond], lat.cuda(), WF, 7.5, use_graph=True)
        s.run(1)
        before = _native.launch_count
        with torch.no_grad():
            unet(s._unet_in, s._params[2:3], encoder_hidden_states=s._ctx)
        unet_launches = _native.launch_count - before
        assert s.native_launches_per_step == unet_launches + 2
        # every CUDA kernel of an eager step beyond the UNet's own is one of the two sampler kernels
        eager = PwWSampler(unet, _setup(cfg, SAMPLERS[name], "cuda")[2], [cond], [uncond], lat.cuda(), WF, 7.5,
                           use_graph=False)
        eager.run(1)
        from torch.profiler import ProfilerActivity, profile

        def kernels(fn):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            return [e.name for e in prof.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name
                    and "Memset" not in e.name]
        with torch.no_grad():
            step_k = kernels(eager._step_body)
            unet_k = kernels(lambda: unet(eager._unet_in, eager._params[2:3], encoder_hidden_states=eager._ctx))
    finally:
        P.unpatch_all()
    extra = list(step_k)
    for k in unet_k:
        extra.remove(k)
    assert sorted("update" if "sampler_update" in k else "input" if "sampler_input" in k else k for k in extra) == \
        ["input", "update"], extra
