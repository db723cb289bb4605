"""ControlNet on the GPU.

Kernel: `pww_control_inject_{f16,bf16}` is bitwise `skip + (r * s)` in torch (the product rounded to the element type)
at the SD1.5, SD2.1 and tiny residual shapes, m = 1, 2, 8, for rows = B and rows = B / 2 (guess mode, the uncond rows
untouched).  Loop: `PwWSampler(controlnet=...)` with the tiny UNet and ControlNet against `reference_controlnet_loop`
(rel RMSE < 3e-2, the bar of the other loop tests), the launch accounting of the two graphs, the guidance window,
guess mode, batching and the public API."""
import math

import pytest
import torch
from PIL import Image

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle.controlnet_loop import reference_controlnet_loop
from paint_with_words_sd_b200 import _native, fused_ops
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.controlnet import build_controlnet, residual_shapes
from paint_with_words_sd_b200.pipeline import PwWSampler, control_scales
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests.fixtures import SETTINGS, color_map_image

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = {"sd15": residual_shapes(UNetConfig.sd15(), 64), "sd21": residual_shapes(UNetConfig.sd21(), 96),
          "tiny": residual_shapes(UNetConfig.tiny(), 16)}


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _case(shapes, B, rows, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    dst = [_cl((torch.randn(B, *s, generator=g) * 2).to(dtype).cuda()) for s in shapes]
    res = [_cl((torch.randn(rows, *s, generator=g) * 3).to(dtype).cuda()) for s in shapes]
    scales = (torch.rand(len(shapes), rows, generator=g) * 2 - 0.5).cuda()
    return dst, res, scales


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("m", [1, 2, 8])
@pytest.mark.parametrize("guess", [False, True])
def test_inject_is_bitwise_torch(dtype, shape, m, guess):
    B = 2 * m
    rows = m if guess else B
    dst, res, scales = _case(SHAPES[shape], B, rows, dtype, seed=m + 17 * guess)
    ref = [d.clone() for d in dst]
    for k, (d, r) in enumerate(zip(ref, res)):
        d[:rows] = d[:rows] + (r * scales[k].view(rows, 1, 1, 1)).to(dtype)    # r * s in fp32, rounded to dtype
    before = [d.clone() for d in dst]
    n0 = _native.launch_count
    fused_ops.control_inject(dst, res, scales)
    torch.cuda.synchronize()
    assert _native.launch_count - n0 == 1
    for k, (d, e) in enumerate(zip(dst, ref)):
        assert torch.equal(d.view(torch.int16), e.view(torch.int16)), (k, (d.float() - e.float()).abs().max().item())
        if guess:
            assert torch.equal(d[rows:].view(torch.int16), before[k][rows:].view(torch.int16)), k


@pytest.mark.parametrize("dtype", DTYPES)
def test_inject_without_scales_is_the_plain_add(dtype):
    dst, res, _ = _case(SHAPES["tiny"], 4, 4, dtype, seed=3)
    ref = [d + r for d, r in zip(dst, res)]
    fused_ops.control_inject(dst, res, None)
    torch.cuda.synchronize()
    for d, e in zip(dst, ref):
        assert torch.equal(d.view(torch.int16), e.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# the loop
# ---------------------------------------------------------------------------------------------------------------------
SIZE, STEPS = 128, 4
WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()     # noqa: E731
TOL = 3e-2


def _scheduler(steps=STEPS):
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(steps)
    return sch


def _encode(cfg, name, device, chunks=1, prompt_repeat=1):
    s = SETTINGS[name]
    _, _, cond, uncond = C._encode_text_color_inputs(
        RandomTextEncoder(cfg.cross_attention_dim).to(device), SimpleWordTokenizer(), device,
        color_map_image(name, SIZE), dict(s["ctx"]), " ".join([s["prompt"]] * prompt_repeat), "",
        max_prompt_chunks=chunks)
    return cond, uncond


def _latents(i, sch, size=SIZE):
    return torch.randn(1, 4, size // 8, size // 8, generator=torch.manual_seed(i)) * sch.init_noise_sigma


def _hint(i, size=SIZE):
    """A scribble-like hint: a few bright rectangles on black."""
    g = torch.Generator().manual_seed(100 + i)
    img = torch.zeros(1, 3, size, size)
    for _ in range(4):
        y, x = torch.randint(0, size - 32, (2,), generator=g).tolist()
        img[:, :, y:y + 32, x:x + 24] = torch.rand(3, 1, 1, generator=g)
    return img


def _rel_rmse(a, b):
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


def _unpatch(unet):
    cls = attention_modules(unet)[0].__class__
    if "__call__" in cls.__dict__:
        delattr(cls, "__call__")


def _reference(cfg, weight=1.0, guess=False, start=0.0, end=1.0, chunks=1, prompt_repeat=1, inpaint=False):
    unet, net = build_unet(cfg, seed=0), build_controlnet(UNetConfig.tiny(), seed=1)
    sch = _scheduler()
    cond, uncond = _encode(cfg, "aurora", "cpu", chunks, prompt_repeat)
    extra = _extra() if inpaint else None
    try:
        oracle_loop.patch_with_oracle(unet)
        return reference_controlnet_loop(unet, net, sch, cond, uncond, _latents(0, sch), WF, _hint(0), 7.5, weight,
                                         guess, start, end, extra_input=extra)
    finally:
        _unpatch(unet)


def _extra():
    g = torch.Generator().manual_seed(9)
    mask = (torch.rand(1, 1, SIZE // 8, SIZE // 8, generator=g) > 0.5).float()
    return torch.cat([mask, torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=g)], 1)


def _gpu(cfg, dtype=torch.float16, use_graph=True, weight=1.0, guess=False, start=0.0, end=1.0, chunks=1,
         prompt_repeat=1, inpaint=False, controlnet=True, net=None):
    unet = build_unet(cfg, seed=0, dtype=dtype, device="cuda")
    if controlnet and net is None:
        net = build_controlnet(UNetConfig.tiny(), seed=1, dtype=dtype, device="cuda")
    sch = _scheduler()
    cond, uncond = _encode(cfg, "aurora", "cuda", chunks, prompt_repeat)
    kw = dict(controlnet=net, control_image=_hint(0), controlnet_conditioning_scale=weight, guess_mode=guess,
              control_guidance_start=start, control_guidance_end=end) if controlnet else {}
    P.patch_unet(unet)
    try:
        s = PwWSampler(unet, sch, [cond], [uncond], _latents(0, sch).cuda(), WF, 7.5, use_graph=use_graph,
                       extra_input=_extra().cuda() if inpaint else None, **kw)
        out = s.run().float().cpu()
    finally:
        P.unpatch_all()
    return out, s


CASES = {
    "graph": dict(),
    "eager": dict(use_graph=False),
    "guess": dict(guess=True, weight=0.8),
    "window": dict(start=0.25, end=0.75),
    "inpaint": dict(inpaint=True),
    "two_chunks": dict(chunks=2, prompt_repeat=3),
    "bf16": dict(dtype=torch.bfloat16),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_sampler_matches_the_reference_loop(case):
    kw = CASES[case]
    cfg = UNetConfig.tiny(in_channels=9 if kw.get("inpaint") else 4)
    ref_kw = {k: v for k, v in kw.items() if k not in ("use_graph", "dtype")}
    ref = _reference(cfg, **ref_kw)
    out, s = _gpu(cfg, **kw)
    if kw.get("chunks"):
        assert s._ctx["CONTEXT_TENSOR"].shape[1] == 154
    assert torch.isfinite(out).all()
    err = _rel_rmse(out, ref)
    assert err < TOL, (case, err)


def test_control_changes_the_result():
    cfg = UNetConfig.tiny()
    with_control, _ = _gpu(cfg)
    without, _ = _gpu(cfg, controlnet=False)
    assert _rel_rmse(with_control, without) > TOL


class _Counting:
    """Wraps a ControlNet's forward: counts calls and records the batch it sees."""

    def __init__(self, net):
        self.calls, self.batches = 0, []
        self._forward = net.forward

        def forward(sample, *a, **k):
            self.calls += 1
            self.batches.append(int(sample.shape[0]))
            return self._forward(sample, *a, **k)
        net.forward = forward


@pytest.mark.parametrize("use_graph", [False, True])
def test_closed_window_is_the_plain_sampler_bit_for_bit(use_graph):
    cfg = UNetConfig.tiny()
    net = build_controlnet(cfg, seed=1, dtype=torch.float16, device="cuda")
    counter = _Counting(net)
    got, s = _gpu(cfg, use_graph=use_graph, start=0.9, end=0.95, net=net)
    plain, p = _gpu(cfg, use_graph=use_graph, controlnet=False)
    assert counter.calls == 0
    assert torch.equal(got, plain)
    if use_graph:
        assert s.native_launches_per_step is None and True not in s._graphs
        assert s.native_launches_per_step_without_control == p.native_launches_per_step


def test_launch_accounting_in_and_out_of_the_window():
    """In the window: the plain step + the ControlNet's launches + ONE injection launch; outside it: the plain step."""
    cfg = UNetConfig.tiny()
    net = build_controlnet(cfg, seed=1, dtype=torch.float16, device="cuda")
    _, s = _gpu(cfg, start=0.0, end=0.5, net=net)
    _, plain = _gpu(cfg, controlnet=False)
    P.patch_unet(net)
    try:
        x = torch.randn(2, 4, SIZE // 8, SIZE // 8, device="cuda", dtype=torch.float16)
        before = _native.launch_count
        net(x, torch.tensor([500.0], device="cuda"), encoder_hidden_states=s._control_ctx,
            controlnet_cond_embedding=s._hints[0])
        net_launches = _native.launch_count - before
    finally:
        P.unpatch_all()
    assert net_launches > 0
    assert s.native_launches_per_step == plain.native_launches_per_step + net_launches + 1
    assert s.native_launches_per_step_without_control == plain.native_launches_per_step
    assert s._control_active == [True, True, True, False]


def test_guess_mode_runs_the_controlnet_on_the_cond_rows_only():
    cfg = UNetConfig.tiny()
    net = build_controlnet(cfg, seed=1, dtype=torch.float16, device="cuda")
    counter = _Counting(net)
    _gpu(cfg, use_graph=False, guess=True, net=net)
    assert counter.batches == [1] * STEPS
    counter = _Counting(net)
    _gpu(cfg, use_graph=False, guess=False, net=net)
    assert counter.batches == [2] * STEPS


def test_batched_images_with_their_own_hints_and_weights_match_solo_runs():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    net = build_controlnet(cfg, seed=1, dtype=torch.float16, device="cuda")
    names, weights = ["aurora", "cat_dog"], [1.0, 0.6]
    P.patch_unet(unet)
    try:
        sch = _scheduler()
        enc = [_encode(cfg, n, "cuda") for n in names]
        lat = torch.cat([_latents(i, sch) for i in range(2)], 0).cuda()
        batch = PwWSampler(unet, sch, [c for c, _ in enc], [u for _, u in enc], lat, WF, 7.5, controlnet=net,
                           control_image=[_hint(0), _hint(1)], controlnet_conditioning_scale=weights).run().float().cpu()
        solo = []
        for i in range(2):
            sch = _scheduler()
            solo.append(PwWSampler(unet, sch, [enc[i][0]], [enc[i][1]], _latents(i, sch).cuda(), WF, 7.5,
                                   controlnet=net, control_image=_hint(i),
                                   controlnet_conditioning_scale=weights[i]).run().float().cpu())
    finally:
        P.unpatch_all()
    for i in range(2):
        d = (batch[i] - solo[i][0]).abs().max().item()
        assert torch.isfinite(batch[i]).all() and d <= 2e-2 * solo[i].abs().max().item(), (i, d)


def _pil_hint(i, size):
    a = (_hint(i, size)[0].permute(1, 2, 0).numpy() * 255).round().astype("uint8")
    return Image.fromarray(a)


def test_public_api_with_a_controlnet():
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    net = P.pww_load_controlnet("synthetic:tiny", device="cuda:0")
    a, c = SETTINGS["aurora"], SETTINGS["cat_dog"]
    entries = [
        dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", 128), input_prompt=a["prompt"], seed=0,
             control_image=_pil_hint(0, 128)),
        dict(color_context=c["ctx"], color_map_image=color_map_image("cat_dog", 128), input_prompt=c["prompt"], seed=1,
             control_image=_pil_hint(1, 128), controlnet_conditioning_scale=0.5),
    ]
    try:
        got = P.paint_with_words_batch(entries, num_inference_steps=3, device="cuda:0", preloaded_utils=tools,
                                       return_latents=True, controlnet=net)
        refs = [P.paint_with_words(**dict(e, color_context=dict(e["color_context"])), num_inference_steps=3,
                                   device="cuda:0", preloaded_utils=tools, return_latents=True, controlnet=net)
                for e in entries]
        plain = P.paint_with_words(**dict(entries[0], color_context=dict(a["ctx"]), control_image=None),
                                   num_inference_steps=3, device="cuda:0", preloaded_utils=tools, return_latents=True)
        image = P.paint_with_words(**dict(entries[0], color_context=dict(a["ctx"])), num_inference_steps=2,
                                   device="cuda:0", preloaded_utils=tools, controlnet=net, guess_mode=True,
                                   control_guidance_end=0.5)
        itools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny-inpaint")
        inp = P.paint_with_words_inpaint(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 128),
                                         mask_image=Image.new("L", (128, 128), 255), init_image=_pil_hint(2, 128),
                                         input_prompt=a["prompt"], num_inference_steps=3, device="cuda:0",
                                         preloaded_utils=itools, return_latents=True, controlnet=net,
                                         control_image=_pil_hint(0, 128))
        pipe = P.PaintWithWord_StableDiffusionPipeline(*[tools[i] for i in (0, 2, 3, 1)], controlnet=net)
        out = pipe(a["prompt"], color_map_image=color_map_image("aurora", 128), color_context=dict(a["ctx"]),
                   num_inference_steps=3, control_image=_pil_hint(0, 128), output_type="latent")
    finally:
        P.unpatch_all()
    for i, (x, ref) in enumerate(zip(got, refs)):
        d = (x.float() - ref.float()).abs().max().item()
        assert torch.isfinite(x).all() and d <= 2e-2 * ref.abs().max().item(), (i, d)
    assert _rel_rmse(refs[0].float().cpu(), plain.float().cpu()) > TOL
    assert image.size == (128, 128)
    assert tuple(inp.shape) == (1, 4, 16, 16) and torch.isfinite(inp).all()
    assert torch.allclose(out.images.float(), refs[0].float(), rtol=0, atol=2e-2 * refs[0].abs().max().item())
