"""Masked img2img on the GPU: `pww_sampler_update_masked` bitwise against the same step written as torch fp32 ops, the
all-ones and all-zeros masks against the unmasked kernels, batch and position invariance; PwWSampler against
`mask_blend_loop` on the CPU; graphs, launch counts and the public API."""
import functools
import math

import pytest
import torch
from PIL import Image

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle import mask_blend_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.pipeline import _BETA, PwWSampler, _dtype_code, ancestral_noise
from paint_with_words_sd_b200.scheduler import (FORM_COLUMNS, DPMSolverMultistepScheduler,
                                                EulerAncestralDiscreteScheduler, EulerDiscreteScheduler,
                                                LMSDiscreteScheduler)
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests.fixtures import SETTINGS, color_map_image
from tests.test_samplers_gpu import _WithNoise
from tests.test_t2i_adapter_gpu import _pil_hint

pytestmark = pytest.mark.gpu
WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
SAMPLERS = {"lms": LMSDiscreteScheduler, "euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler,
            "dpmpp_2m": DPMSolverMultistepScheduler,
            "dpmpp_2m_karras": functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=True)}


def _scheduler(name, steps, prediction_type="epsilon"):
    sch = SAMPLERS[name](**KW, prediction_type=prediction_type)
    sch.set_timesteps(steps)
    return sch


def _contexts(m):
    g = torch.Generator().manual_seed(0)
    return ([{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)],
            [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)])


# ---- the kernel ------------------------------------------------------------------------------------------------------
def _outputs(m, h, w, dtype, layout, steps, seed):
    """`steps` UNet outputs [2m, 4, h, w] in `dtype` and `layout`."""
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


def _mask(kind, m, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "ones":
        return torch.ones(m, 1, h, w)
    if kind == "zeros":
        return torch.zeros(m, 1, h, w)
    if kind == "soft":                      # soft values, with exact 0 and 1 among them
        return (torch.rand(m, 1, h, w, generator=g) * 1.4 - 0.2).clamp(0, 1)
    return (torch.rand(m, 1, h, w, generator=g) > 0.5).float()


class _Run:
    """The sampler state one kernel run needs (step rows with sigma', history, noise, guidance, phi, init latents,
    init noise and mask) from a PwWSampler over m images that is never stepped."""

    def __init__(self, name, m, h, w, phis, steps, mask="binary", seed=0):
        g = torch.Generator().manual_seed(seed + 17)
        conds, unconds = _contexts(m)
        self.init = torch.randn(m, 4, h, w, generator=g).cuda()
        self.z0 = torch.randn(m, 4, h, w, generator=g).cuda()
        self.mask = _mask(mask, m, h, w, seed).cuda()
        sch = _scheduler(name, steps + 2)
        ts = sch.timesteps[2:]
        self.lat0 = sch.add_noise(self.init, self.z0, ts[:1])
        self.s = PwWSampler(torch.nn.Linear(1, 1).cuda(), sch, conds, unconds, self.lat0, WF,
                            [7.5 - 1.5 * (i % 4) for i in range(m)], use_graph=False,
                            noise_seed=list(range(100, 100 + m)), guidance_rescale=phis, timesteps=ts,
                            init_latents=self.init, init_noise=self.z0, inpaint_mask=self.mask)
        self.phi = torch.tensor(phis, dtype=torch.float32, device="cuda")
        self.rescale = any(phis)
        self.m, self.h, self.w = m, h, w
        self.sn = self.s._form + len(FORM_COLUMNS)

    def _args(self, eps, lat, hist, p):
        s = self.s
        return (eps.data_ptr(), _dtype_code(eps.dtype), *eps.stride(), lat.data_ptr(), hist.data_ptr(), s._hist_len,
                None if s._noise is None else s._noise.data_ptr(), s._gscale.data_ptr(), p[_BETA:].data_ptr(),
                p[s._form:].data_ptr())

    def launch(self, i, eps, lat, hist, masked=True, stats=None):
        """Step i in place on (lat, hist): the masked update, or with masked=False the unmasked kernel of the same
        rescale setting."""
        m, h, w = self.m, self.h, self.w
        L = _native.lib()
        p = self.s._rows[i].clone()
        args = self._args(eps, lat, hist, p)
        phi = self.phi.data_ptr() if self.rescale else None
        st = None if stats is None else stats.data_ptr()
        if masked:
            _native.check(L.pww_sampler_update_masked(*args, phi, st, self.init.data_ptr(), self.z0.data_ptr(),
                                                      self.mask.data_ptr(), p[self.sn:].data_ptr(), m, h, w, None),
                          "pww_sampler_update_masked")
        elif self.rescale:
            _native.check(L.pww_sampler_update_rescale(*args, phi, st, m, h, w, None), "pww_sampler_update_rescale")
        else:
            _native.check(L.pww_sampler_update(*args, m, h, w, None), "pww_sampler_update")

    def kernel(self, outs, masked=True):
        """The native run over every step: (latents, history, per-step stats [steps, m, 3] or None)."""
        lat, hist = self.lat0.clone(), torch.zeros_like(self.s._derivs)
        stats = []
        for i, eps in enumerate(outs):
            st = torch.full((self.m, 3), float("nan"), device="cuda") if self.rescale else None
            self.launch(i, eps, lat, hist, masked, st)
            stats.append(st)
        torch.cuda.synchronize()
        return lat, hist, (torch.stack(stats) if self.rescale else None)

    def torch_ops(self, outs, ks):
        """The same run as torch fp32 ops in the kernel's order, with the kernel's k of every step."""
        s, m = self.s, self.m
        lat, ring = self.lat0.clone(), torch.zeros_like(s._derivs)
        L = ring.shape[0]
        for i, eps in enumerate(outs):
            r = [float(v) for v in s._rows[i].tolist()]
            alpha, a, b, gamma, slot, nrow = r[s._form:self.sn]
            sigma_next = r[self.sn]
            beta = r[3:7]
            e = eps.float()
            e = e[m:] + s._gscale * (e[:m] - e[m:])
            if ks is not None:
                e = torch.where(self.phi.view(m, 1, 1, 1) != 0, ks[i].view(m, 1, 1, 1) * e, e)
            q = b * e if a == 0 else a * lat + b * e
            ring[int(slot)].copy_(q)
            acc = beta[0] * q
            for j in range(1, L):
                acc = acc + beta[j] * ring[(int(slot) - j) % L]
            out = lat + acc if alpha == 1 else alpha * lat + acc
            if gamma != 0 and s._noise is not None:
                out = out + gamma * s._noise[int(nrow)]
            lat = self.mask * out + (1 - self.mask) * (self.init + self.z0 * sigma_next)
        return lat, ring


def _kernel_case(name, m, hw, dtype, layout, phis, steps=4, mask="binary"):
    h, w = hw
    run = _Run(name, m, h, w, phis, steps, mask, seed=h * 100 + w)
    outs = _outputs(m, h, w, dtype, layout, steps, seed=h * 7 + w)
    lat, hist, stats = run.kernel(outs)
    assert torch.isfinite(lat).all()
    want_lat, want_hist = run.torch_ops(outs, None if stats is None else stats[:, :, 2])
    assert torch.equal(lat, want_lat)
    assert torch.equal(hist, want_hist)
    if stats is not None:
        # the statistics depend on the UNet outputs only: the unmasked rescale kernel's rows, bit for bit
        _, _, plain_stats = run.kernel(outs, masked=False)
        assert torch.equal(stats, plain_stats)
    return run, outs, lat


SIZES = [(8, 8), (13, 7), (64, 64), (96, 96), (128, 128)]


@pytest.mark.parametrize("rescale", [False, True], ids=["cfg", "rescale"])
@pytest.mark.parametrize("name", list(SAMPLERS))
@pytest.mark.parametrize("hw", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_masked_kernel_every_sampler_and_size(name, hw, rescale):
    _kernel_case(name, 3, hw, torch.float16, "channels_last", [0.7, 0.0, 1.0] if rescale else [0.0] * 3)


@pytest.mark.parametrize("rescale", [False, True], ids=["cfg", "rescale"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("layout", ["channels_last", "contiguous", "strided"])
@pytest.mark.parametrize("hw", [(13, 7), (64, 64)], ids=["13x7", "64x64"])
def test_masked_kernel_every_dtype_and_layout(dtype, layout, hw, rescale):
    _kernel_case("euler_a", 2, hw, dtype, layout, [0.0, 0.7] if rescale else [0.0, 0.0])


@pytest.mark.parametrize("m", [1, 3, 8])
@pytest.mark.parametrize("rescale", [False, True], ids=["cfg", "rescale"])
def test_masked_kernel_soft_mask_and_batch_sizes(m, rescale):
    phis = [0.7 if (rescale and i % 2 == 0) else 0.0 for i in range(m)]
    _kernel_case("dpmpp_2m", m, (96, 96), torch.bfloat16, "channels_last", phis, mask="soft")


@pytest.mark.parametrize("rescale", [False, True], ids=["cfg", "rescale"])
@pytest.mark.parametrize("name", ["lms", "euler_a", "dpmpp_2m"])
@pytest.mark.parametrize("hw", [(64, 64), (13, 7)], ids=["64x64", "13x7"])
def test_all_ones_mask_is_the_unmasked_update(name, hw, rescale):
    h, w = hw
    run = _Run(name, 3, h, w, [0.7, 0.0, 0.3] if rescale else [0.0] * 3, 4, mask="ones")
    outs = _outputs(3, h, w, torch.float16, "channels_last", 4, seed=1)
    lat, hist, stats = run.kernel(outs)
    plain_lat, plain_hist, plain_stats = run.kernel(outs, masked=False)
    assert torch.equal(lat, plain_lat) and torch.equal(hist, plain_hist)
    if rescale:
        assert torch.equal(stats, plain_stats)


@pytest.mark.parametrize("rescale", [False, True], ids=["cfg", "rescale"])
@pytest.mark.parametrize("name", ["lms", "euler_a", "dpmpp_2m_karras"])
def test_all_zeros_mask_is_the_noised_init(name, rescale):
    """From the same state, a masked step with M = 0 writes the unmasked step's history entry and leaves the latents
    at add_noise(init, z, sigma'); the last step leaves init itself."""
    h, w, steps = 64, 64, 4
    run = _Run(name, 2, h, w, [0.7, 0.0] if rescale else [0.0, 0.0], steps, mask="zeros")
    outs = _outputs(2, h, w, torch.float32, "contiguous", steps, seed=2)
    lat, hist = run.lat0.clone(), torch.zeros_like(run.s._derivs)
    sch = run.s.scheduler
    for i, eps in enumerate(outs):
        plain_lat, plain_hist = lat.clone(), hist.clone()
        run.launch(i, eps, plain_lat, plain_hist, masked=False)
        run.launch(i, eps, lat, hist)
        assert torch.equal(hist, plain_hist), i
        if i + 1 < steps:
            assert torch.equal(lat, sch.add_noise(run.init, run.z0, run.s.timesteps[i + 1:i + 2])), i
        lat = plain_lat              # the next step starts from the unmasked state
    run.launch(steps - 1, outs[-1], lat, hist)
    assert torch.equal(lat, run.init)


@pytest.mark.parametrize("rescale", [False, True], ids=["cfg", "rescale"])
@pytest.mark.parametrize("hw", [(64, 64), (96, 96), (13, 7)], ids=["64x64", "96x96", "13x7"])
def test_masked_kernel_is_batch_and_position_invariant(hw, rescale):
    """Image i's latents and history are the same bits alone, in a batch of 3 or 8 and at any position."""
    h, w = hw
    steps, m = 3, 8
    phis = [0.7, 0.0, 1.0, 0.3, 0.5, 0.9, 0.0, 0.2] if rescale else [0.0] * m
    run = _Run("lms", m, h, w, phis, steps)
    outs = _outputs(m, h, w, torch.float16, "channels_last", steps, seed=5)
    lat, hist, _ = run.kernel(outs)

    def subset(idx):
        sub = _Run("lms", len(idx), h, w, [phis[i] for i in idx], steps)
        sub.lat0, sub.init, sub.z0 = run.lat0[idx].clone(), run.init[idx].clone(), run.z0[idx].clone()
        sub.mask = run.mask[idx].clone()
        sub.s._gscale = run.s._gscale[idx].contiguous()
        rows = torch.cat([torch.as_tensor(idx), torch.as_tensor(idx) + m]).cuda()
        return sub.kernel([o[rows].contiguous(memory_format=torch.channels_last) for o in outs])
    for idx in ([2], [5], [0], [6, 2, 4], [7, 1, 3]):
        sl, sh, _ = subset(idx)
        assert torch.equal(sl, lat[idx]), idx
        assert torch.equal(sh, hist[:, idx]), idx


# ---- the sampler against the reference loop ------------------------------------------------------------------------
SIZE, STEPS, START = 128, 6, 2


def _inputs(cfg, name, device, prediction_type="epsilon"):
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim)
    s = SETTINGS["aurora"]
    _, _, cond, uncond = C._encode_text_color_inputs(enc.to(device), tok, device, color_map_image("aurora", SIZE),
                                                     dict(s["ctx"]), s["prompt"], "")
    sch = _scheduler(name, STEPS, prediction_type)
    g = torch.Generator().manual_seed(3)
    init = torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=g)
    z = torch.randn(init.shape, generator=g)
    mask = torch.zeros(1, 1, SIZE // 8, SIZE // 8)
    mask[..., :, SIZE // 16:] = 1                # the right half is repainted
    ts = sch.timesteps[START:]
    return cond, uncond, sch, init, z, mask, ts


CASES = [(n, "epsilon", 0.0) for n in SAMPLERS] + [("euler", "v_prediction", 0.7), ("dpmpp_2m", "v_prediction", 0.7)]


def _reference(case):
    name, pred, phi = case
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0)
    try:
        oracle_loop.patch_with_oracle(unet)
        cond, uncond, sch, init, z, mask, ts = _inputs(cfg, name, "cpu", pred)
        lat = sch.add_noise(init, z, ts[:1])
        if name == "euler_a":
            sch = _WithNoise(sch, ancestral_noise([0], (1, 4, SIZE // 8, SIZE // 8), len(ts))[:, 0])
        return mask_blend_loop.reference_mask_blend_loop(unet, sch, cond, uncond, lat, WF, init, z, mask, 7.5,
                                                         guidance_rescale=phi, timesteps=ts), init, mask
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")


def _native_run(case, use_graph=True, masked=True):
    name, pred, phi = case
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    cond, uncond, sch, init, z, mask, ts = _inputs(cfg, name, "cuda", pred)
    blend = dict(init_latents=init.cuda(), init_noise=z.cuda(), inpaint_mask=mask.cuda()) if masked else {}
    try:
        P.patch_unet(unet)
        s = PwWSampler(unet, sch, [cond], [uncond], sch.add_noise(init, z, ts[:1]).cuda(), WF, 7.5,
                       use_graph=use_graph, noise_seed=0, guidance_rescale=phi, timesteps=ts, **blend)
        return s.run().float().cpu(), s
    finally:
        P.unpatch_all()


@pytest.mark.parametrize("case", CASES, ids=[f"{n}-{p}-{phi}" for n, p, phi in CASES])
def test_masked_sampler_matches_reference_loop(case):
    ref, init, mask = _reference(case)
    out, _ = _native_run(case)
    d = (out - ref).abs().max().item()
    assert torch.isfinite(out).all() and d <= 2e-2 * ref.abs().max().item(), d
    keep = (mask == 0).expand_as(out)
    assert torch.equal(out[keep], init[keep])
    assert not torch.allclose(out[~keep], init[~keep])


@pytest.mark.parametrize("name", ["lms", "euler_a", "dpmpp_2m_karras"])
def test_graph_and_eager_give_the_same_bits(name):
    case = (name, "epsilon", 0.7)
    assert torch.equal(_native_run(case, use_graph=True)[0], _native_run(case, use_graph=False)[0])


class _TorchUNet(torch.nn.Module):
    """A UNet stand-in made of torch ops only, so a step's native launches are the sampler's own."""

    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(4, 4, 3, padding=1).cuda()

    def forward(self, x, t, encoder_hidden_states=None):
        class _Out:
            sample = torch.tanh(self.conv(x.float()))
        return _Out()


def test_a_masked_step_is_two_native_launches():
    counts = []
    for masked in (False, True):
        for phi in (0.0, 0.7):
            cfg = UNetConfig.tiny()
            cond, uncond, sch, init, z, mask, ts = _inputs(cfg, "dpmpp_2m", "cuda")
            blend = dict(init_latents=init.cuda(), init_noise=z.cuda(), inpaint_mask=mask.cuda()) if masked else {}
            s = PwWSampler(_TorchUNet(), sch, [cond], [uncond], sch.add_noise(init, z, ts[:1]).cuda(), WF, 7.5,
                           guidance_rescale=phi, timesteps=ts, **blend)
            s.run(1)
            counts.append(s.native_launches_per_step)
    assert counts == [2, 2, 2, 2]
    # and on the tiny UNet, a masked step launches as many kernels as an unmasked one
    assert _native_run(("lms", "epsilon", 0.0))[1].native_launches_per_step == \
        _native_run(("lms", "epsilon", 0.0), masked=False)[1].native_launches_per_step


# ---- the public API ------------------------------------------------------------------------------------------------
def _half_mask(size=128):
    m = Image.new("L", (size, size), 0)
    m.paste(255, (size // 2, 0, size, size))
    return m


def _public(tools, mask_image, seed=11, **kw):
    """paint_with_words img2img from the global seed `seed`: (latents, init latents, native launches)."""
    a = SETTINGS["aurora"]
    vae, _, _, _, sch = tools
    init_image = _pil_hint(2, 128)
    torch.manual_seed(seed)
    sch.set_timesteps(6)
    init = PL._img2img_latents(vae, sch, init_image, 6, 0.75, "cuda:0")[2]
    before = _native.launch_count
    torch.manual_seed(seed)
    out = P.paint_with_words(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 128),
                             input_prompt=a["prompt"], num_inference_steps=6, device="cuda:0", preloaded_utils=tools,
                             weight_function=WF, init_image=init_image, strength=0.75, mask_image=mask_image,
                             return_latents=True, **kw)
    return out, init, _native.launch_count - before


def test_public_masked_img2img_keeps_the_init_latents_outside_the_mask():
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    try:
        lat, init, launches = _public(tools, _half_mask())
        white, _, white_launches = _public(tools, Image.new("L", (128, 128), 255))
        plain, _, plain_launches = _public(tools, None)
    finally:
        P.unpatch_all()
    assert torch.equal(lat[..., :8], init[..., :8]) and not torch.allclose(lat[..., 8:], init[..., 8:])
    assert torch.equal(white, plain)
    assert launches == white_launches == plain_launches


@pytest.mark.parametrize("unit", ["controlnet", "adapter", "attention_maps"])
def test_public_masked_img2img_with_units_and_maps(unit):
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    if unit == "controlnet":
        kw = dict(controlnet=P.pww_load_controlnet("synthetic:tiny", device="cuda:0", seed=1),
                  control_image=_pil_hint(0, 128))
    elif unit == "adapter":
        kw = dict(controlnet=P.pww_load_adapter("synthetic:tiny:full192", device="cuda:0"),
                  control_image=_pil_hint(1, 128))
    else:
        kw = dict(return_attention_maps=True)
    try:
        got, init, launches = _public(tools, _half_mask(), **kw)
        white, _, white_launches = _public(tools, Image.new("L", (128, 128), 255), **kw)
        plain, _, plain_launches = _public(tools, None, **kw)
    finally:
        P.unpatch_all()
    if unit == "attention_maps":
        (got, maps), (white, wmaps), (plain, pmaps) = got, white, plain
        assert torch.equal(wmaps.maps, pmaps.maps) and torch.isfinite(maps.maps).all()
    assert torch.equal(got[..., :8], init[..., :8])
    assert torch.equal(white, plain)
    assert launches == white_launches == plain_launches


def test_pipeline_class_mask_image():
    a = SETTINGS["aurora"]
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    vae, unet, enc, tok, sch = tools
    try:
        pipe = P.PaintWithWord_StableDiffusionPipeline(vae, enc, tok, unet, scheduler=sch)
        outs = []
        for mask in (_half_mask(), None):
            torch.manual_seed(5)
            outs.append(pipe(a["prompt"], color_map_image=color_map_image("aurora", 128),
                             color_context=dict(a["ctx"]), weight_function=WF, num_inference_steps=6,
                             image=_pil_hint(2, 128), eta=0.75, mask_image=mask, output_type="latent").images)
        torch.manual_seed(5)
        pipe.scheduler.set_timesteps(6)
        init = PL._img2img_latents(vae, pipe.scheduler, _pil_hint(2, 128), 6, 0.75, "cuda:0")[2]
        with pytest.raises(ValueError, match="mask_image needs an init_image"):
            pipe(a["prompt"], color_map_image=color_map_image("aurora", 128), color_context=dict(a["ctx"]),
                 num_inference_steps=6, mask_image=_half_mask(), output_type="latent")
    finally:
        P.unpatch_all()
    assert torch.equal(outs[0][..., :8], init[..., :8]) and not torch.equal(outs[0], outs[1])
