"""Full-size UNet parity: the fast route of `unet.py` (native GroupNorm / GEGLU / add+LayerNorm / residual epilogues,
native attention through `inj_forward`, channels-last glue, the batched time projection, the fused QKV / KV weights,
the ControlNet inject and the adapter epilogue) at the production configurations -- SD1.5 at 512 and 256 px,
SD1.5-inpaint, SD2.1 at 768 px -- compared module by module with an fp32 reference of the same weights.

Three routes run on one seeded model:
  * subject: the fp16 / bf16 model E on the fast route (`fused_ops.ENABLED`, `patch_unet` with the library's
    `inj_forward`);
  * baseline: the same E model on the plain PyTorch route with the oracle's attention rounding where an eager E autocast
    rounds -- the code the fast route replaces;
  * reference: an fp32 copy holding exactly E's weights, the plain route, the oracle's attention in fp32, TF32 off (with
    cuDNN's TF32 on, the reference's convolutions would round to the 10 mantissa bits of the fp16 they judge).
Forward hooks record the output of every ResNet block, transformer, down / mid / up block and `conv_out`.  For every
module and for both the relative RMS error and the max absolute error over the reference's RMS (which catches a single
wrong tile row that the RMS averages away), the subject must satisfy

    err_subject <= K * err_baseline + FLOOR[E]

and a failure names the first module, in forward order, that breaks it -- where a broken kernel enters the model.  The
mutation tests at the end show that plausible bugs in the glue are caught at the module where they enter."""
import contextlib
import copy
import gc
import math
import time

import pytest
import torch
import torch.nn.functional as F

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from paint_with_words_sd_b200 import attention, fused_ops
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200 import unet as U
from paint_with_words_sd_b200.pipeline import PwWSampler
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import (CrossAttention, ResnetBlock2D, Transformer2DModel, UNetConfig, build_unet)
from tests.fixtures import SETTINGS, color_map_image

# The bound, from the errors of every case below measured on an H100 80GB HBM3 (700 W power limit).  Over all modules
# of all cases the subject's relative RMS error is at most 0.87x the baseline's and its max error at most 1.13x (fp16)
# / 1.16x (bf16), so K = 1.5 leaves the worst module at 0.75 of the bound.  K = 2 would no longer catch the
# self-attention that drops 16 of 1024 keys where it enters (its relative RMS error is 2.5x the baseline's there).
# FLOOR is about half a unit roundoff of E (2^-11 for fp16, 2^-8 for bf16): it only matters for modules whose
# baseline error is itself below that.
K = 1.5
FLOOR = {torch.float16: 2e-4, torch.bfloat16: 2e-3}
# A reference module output whose RMS falls below this would mean the random model has collapsed (the smallest
# measured is 0.21).
MIN_REF_RMS = 0.05
# Sharpened case: every to_q weight is multiplied by SHARPEN, so that attention at the 1024-key self-attention level is
# peaked: the mean over rows (and heads) of the largest softmax probability must exceed PEAKED.  Measured 0.50 at
# SHARPEN = 16 (0.077 at 6, 0.26 at 10, 0.67 at 24, where the fp16 errors of both routes grow past 5e-2).
SHARPEN = 16.0
PEAKED = 0.4

WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731  (runner.py:104)
ZERO_WF = lambda w, sigma, qk: 0.0                                      # noqa: E731
CONFIGS = {"sd15": UNetConfig.sd15, "sd15_inpaint": UNetConfig.sd15_inpaint, "sd21": UNetConfig.sd21}
DT = {torch.float16: "fp16", torch.bfloat16: "bf16"}
CL = torch.channels_last
F16, BF16 = torch.float16, torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------------
# recording and comparing module outputs
# ---------------------------------------------------------------------------------------------------------------------
def watched_modules(unet):
    """(name, module) of every module whose output is compared, in definition order."""
    kinds = (ResnetBlock2D, Transformer2DModel, U._DownBlock, U._Mid, U._UpBlock)
    return [(n, m) for n, m in unet.named_modules() if isinstance(m, kinds) or n == "conv_out"]


def record_outputs(unet, run, dtype=torch.float32):
    """Runs `run()` with forward hooks on `watched_modules(unet)`; returns ({name: copy of the module's output in
    `dtype`}, in the order the modules finished, and run's result).  Copies, because later ops (the ControlNet inject)
    update skips in place.  A down block's output is its first element (the activation, not the skip list)."""
    rec = {}

    def hook(name):
        def f(mod, args, out):
            t = out[0] if isinstance(out, tuple) else out
            rec[name] = t.detach().to(dtype, copy=True)
        return f

    handles = [m.register_forward_hook(hook(n)) for n, m in watched_modules(unet)]
    try:
        with torch.no_grad():
            result = run()
    finally:
        for h in handles:
            h.remove()
    return rec, result


def errors(x: torch.Tensor, ref: torch.Tensor):
    """(relative RMS error, max absolute error / RMS of ref), in fp64."""
    r = ref.double()
    d = x.double() - r
    rms = r.pow(2).mean().sqrt()
    return (d.pow(2).mean().sqrt() / rms).item(), (d.abs().max() / rms).item()


def compare(subject: dict, baseline: dict, reference: dict, k: float, floor: float):
    """Per module of `reference` (forward order): (name, subject errors, baseline errors).  Returns (rows, first
    violation or None); a violation is (name, metric, subject error, baseline error)."""
    rows, bad = [], None
    for name, ref in reference.items():
        es, eb = errors(subject[name], ref), errors(baseline[name], ref)
        rows.append((name, es, eb))
        for metric, s, b in zip(("rel_rms", "max/rms"), es, eb):
            if bad is None and not s <= k * b + floor:       # `not <=` also catches NaN
                bad = (name, metric, s, b)
    return rows, bad


def check_reference(reference: dict):
    for name, ref in reference.items():
        assert torch.isfinite(ref).all(), f"reference output of {name} is not finite"
        rms = ref.double().pow(2).mean().sqrt().item()
        assert rms > MIN_REF_RMS, f"reference output of {name} has RMS {rms:.3g}: the random model collapsed"


def report(case: str, rows, k: float, floor: float, n: int = 5):
    """Prints the n modules closest to the bound (largest err_subject / (K * err_baseline + FLOOR) of either metric)."""
    def margin(row):
        _, es, eb = row
        return max(s / (k * b + floor) for s, b in zip(es, eb))
    print(f"\n[{case}] worst {n} of {len(rows)} modules (subject rel_rms, max/rms | baseline rel_rms, max/rms):")
    for row in sorted(rows, key=margin, reverse=True)[:n]:
        name, es, eb = row
        print(f"  {name:40s} {es[0]:.3e} {es[1]:.3e} | {eb[0]:.3e} {eb[1]:.3e}  ({margin(row):.2f} of the bound)")


def assert_within_bound(case: str, subject: dict, baseline: dict, reference: dict, dtype):
    assert list(subject) == list(reference) and list(baseline) == list(reference), "module order differs"
    rows, bad = compare(subject, baseline, reference, K, FLOOR[dtype])
    report(case, rows, K, FLOOR[dtype])
    check_reference(reference)
    assert bad is None, (f"{case}: first module out of bound: {bad[0]} ({bad[1]}: subject {bad[2]:.3e} > "
                         f"{K} * baseline {bad[3]:.3e} + {FLOOR[dtype]:g})")


# ---------------------------------------------------------------------------------------------------------------------
# the three routes
# ---------------------------------------------------------------------------------------------------------------------
def _drop_oracle_patch():
    if "__call__" in CrossAttention.__dict__:
        delattr(CrossAttention, "__call__")


@contextlib.contextmanager
def _fast_route(enabled: bool):
    prev = fused_ops.ENABLED
    fused_ops.ENABLED = enabled
    try:
        yield
    finally:
        fused_ops.ENABLED = prev


@contextlib.contextmanager
def _no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def run_subject(unet, run):
    with _fast_route(True):
        try:
            P.patch_unet(unet)
            return record_outputs(unet, run)
        finally:
            P.unpatch_all()


def run_baseline(unet, run, dtype):
    with _fast_route(False):
        try:
            oracle_loop.patch_with_oracle(unet, emulate_dtype=dtype)
            return record_outputs(unet, run)
        finally:
            _drop_oracle_patch()


def run_reference(ref, run):
    with _fast_route(False), _no_tf32():
        try:
            oracle_loop.patch_with_oracle(ref)
            return record_outputs(ref, run)
        finally:
            _drop_oracle_patch()


def three_routes(models, kw_e: dict, kw_ref: dict):
    """Module outputs of one forward `unet(**kw)` on the three routes: kw_e for the E model, kw_ref (the same values in
    fp32) for the reference."""
    subj, _ = run_subject(models.unet, lambda: models.unet(**kw_e))
    base, _ = run_baseline(models.unet, lambda: models.unet(**kw_e), models.dtype)
    ref, _ = run_reference(models.ref, lambda: models.ref(**kw_ref))
    return subj, base, ref


@pytest.fixture(autouse=True)
def _restore_state():
    """Every test leaves the fast-route switch, the self-attention dispatch, the TF32 flags, the class patch and the
    shim's device state as it found them."""
    flags = (fused_ops.ENABLED, attention.SELF_ATTN_IMPL, torch.backends.cuda.matmul.allow_tf32,
             torch.backends.cudnn.allow_tf32)
    yield
    (fused_ops.ENABLED, attention.SELF_ATTN_IMPL, torch.backends.cuda.matmul.allow_tf32,
     torch.backends.cudnn.allow_tf32) = flags
    P.unpatch_all()
    _drop_oracle_patch()
    attention.reset_device_state()


# ---------------------------------------------------------------------------------------------------------------------
# models and inputs
# ---------------------------------------------------------------------------------------------------------------------
class _Models:
    def __init__(self, name, dtype, unet, ref):
        self.name, self.dtype, self.unet, self.ref = name, dtype, unet, ref
        self.cfg = unet.config


_CACHE = {}


def _release():
    _CACHE.clear()
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _host(name: str):
    """The seeded fp32 host model of a configuration, built once while that configuration is in use."""
    if _CACHE.get("host_name") != name:
        _release()
        _CACHE["host"] = build_unet(CONFIGS[name](), seed=0)
        _CACHE["host_name"] = name
    return _CACHE["host"]


def _to_device(host, dtype, sharpen: float = 1.0):
    """(E model on CUDA, fp32 copy of its E-rounded weights on CUDA), both channels-last."""
    m = copy.deepcopy(host)
    if sharpen != 1.0:
        with torch.no_grad():
            for a in U.attention_modules(m):
                a.to_q.weight.mul_(sharpen)
    unet = m.to(device="cuda", dtype=dtype).to(memory_format=CL)
    return unet, copy.deepcopy(unet).float()


def models(name: str, dtype) -> _Models:
    """E model and reference of (configuration, dtype), cached while that pair is in use; the previous pair is freed
    first."""
    hit = _CACHE.get("models")
    if hit is None or (hit.name, hit.dtype) != (name, dtype):
        host = _host(name)
        _CACHE.pop("models", None)
        gc.collect()
        torch.cuda.empty_cache()
        _CACHE["models"] = _Models(name, dtype, *_to_device(host, dtype))
    return _CACHE["models"]


@pytest.fixture(scope="module", autouse=True)
def _module_models():
    """Frees the cached models when the module ends and prints its wall time and peak GPU memory."""
    t0 = time.perf_counter()
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    _release()
    if torch.cuda.is_available():
        print(f"\n[{__name__}] wall {time.perf_counter() - t0:.1f} s, peak GPU memory "
              f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def _scheduler(steps: int):
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(steps)
    return sch


def _round_maps(d: dict, dtype) -> dict:
    """The context dict with every device weight map rounded to `dtype` (kept in fp32: one map for all routes)."""
    return {k: (v.to(dtype).float() if torch.is_tensor(v) and k.startswith("CROSS_ATTENTION_WEIGHT_") and v.is_cuda
                else v) for k, v in d.items()}


def pww_dicts(cfg, size: int, dtype):
    """The paint-with-words (cond, uncond) dicts of the golden `aurora` colour map at image size `size`, built as
    `test_pipeline_gpu._setup` builds them, with the weight maps rounded to dtype."""
    s = SETTINGS["aurora"]
    _, _, cond, uncond = C._encode_text_color_inputs(RandomTextEncoder(cfg.cross_attention_dim).to("cuda"),
                                                     SimpleWordTokenizer(), "cuda", color_map_image("aurora", size),
                                                     dict(s["ctx"]), s["prompt"], "")
    return _round_maps(cond, dtype), uncond


def _with_ctx(d: dict, ctx: torch.Tensor) -> dict:
    return dict(d, CONTEXT_TENSOR=ctx)


class Case:
    """The inputs of one forward: `kw(dtype)` for the E routes, `kw(torch.float32)` for the reference.  Every tensor is
    E-rounded first, so the three routes see the same values."""

    def __init__(self, cfg, latent: int, dtype, context: str, batch: int = None):
        self.cfg, self.dtype = cfg, dtype
        sch = _scheduler(50)
        self.t, self.sigma = sch.timesteps[0], sch.sigmas[0]              # the first (largest) LMS sigma
        cond, uncond = pww_dicts(cfg, latent * 8, dtype)
        ctx = {"cond": cond["CONTEXT_TENSOR"].to(dtype), "uncond": uncond["CONTEXT_TENSOR"].to(dtype)}
        self.stacked = torch.cat([ctx["cond"], ctx["uncond"]], 0)
        self.cond = dict(cond, SIGMA=self.sigma, WEIGHT_FUNCTION=WF)
        self.context = context
        batch = batch or (1 if context == "pww" else 2)
        g = torch.Generator().manual_seed(7)
        self.sample = torch.randn(batch, cfg.in_channels, latent, latent, generator=g).to(dtype).float().cuda()
        self.extra = {}                           # further forward kwargs: {name: E tensor or list of E tensors}
        self.control_scales = None                # fp32 [13, rows] CONTROL_SCALES of the "scaled" context

    def context_for(self, dtype):
        if self.context == "tensor":
            return self.stacked.to(dtype)
        if self.context == "pww":
            return _with_ctx(self.cond, self.stacked[:1].to(dtype))
        # "scaled": the stacked contexts in the pww dict with a zero weight function (no bias) and CONTROL_SCALES
        return dict(_with_ctx(self.cond, self.stacked.to(dtype)), WEIGHT_FUNCTION=ZERO_WF,
                    CONTROL_SCALES=self.control_scales)

    def kw(self, dtype):
        def cast(v):
            if isinstance(v, (list, tuple)):
                return [cast(t) for t in v]
            return v if dtype != torch.float32 else v.float()
        kw = {"sample": self.sample, "timestep": self.t, "encoder_hidden_states": self.context_for(dtype)}
        kw.update({k: cast(v) for k, v in self.extra.items()})
        return kw


def _rand(shape, g, dtype, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda().contiguous(memory_format=CL)


def skip_shapes(cfg, latent: int):
    """[C, h, w] of the 12 skips (conv_in, each encoder layer, each downsampler) and of the mid block's output."""
    ch, n = cfg.block_out_channels, cfg.layers_per_block
    shapes, s = [(ch[0], latent, latent)], latent
    for i, c in enumerate(ch):
        shapes += [(c, s, s)] * n
        if i < len(ch) - 1:
            s = (s + 1) // 2
            shapes.append((c, s, s))
    return shapes, (ch[-1], s, s)


def run_case(m: _Models, case: Case):
    return three_routes(m, case.kw(m.dtype), case.kw(torch.float32))


def _id(v):
    return DT.get(v, str(v))


# ---------------------------------------------------------------------------------------------------------------------
# 1. single forwards at the production configurations
# ---------------------------------------------------------------------------------------------------------------------
_SHAPES = [("sd15", 64, F16), ("sd15", 32, F16), ("sd15", 64, BF16), ("sd15", 32, BF16), ("sd15_inpaint", 64, F16),
           ("sd21", 96, BF16), ("sd21", 96, F16)]
FORWARD_CASES = [(n, lat, dt, ctx, impl) for n, lat, dt in _SHAPES for ctx in ("tensor", "pww")
                 for impl in ("auto", "native")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,latent,dtype,context,impl", FORWARD_CASES,
                         ids=[f"{n}-{lat * 8}px-{_id(dt)}-{c}-{i}" for n, lat, dt, c, i in FORWARD_CASES])
def test_full_size_forward_within_bound(name, latent, dtype, context, impl):
    """One forward of the production UNet: a batch-2 plain-context forward (stacked cond + uncond contexts) or the
    batch-1 cond forward with the paint-with-words dict at the first LMS sigma, with self-attention dispatched as shipped
    ("auto": native up to 1024 keys, the library above) or forced native (4096 and 9216 keys inside the model)."""
    m = models(name, dtype)
    case = Case(m.cfg, latent, dtype, context)
    attention.SELF_ATTN_IMPL = impl
    subj, base, ref = run_case(m, case)
    assert_within_bound(f"{name} {latent * 8}px {_id(dtype)} {context} {impl}", subj, base, ref, dtype)


# ---------------------------------------------------------------------------------------------------------------------
# 2. a short full-size loop
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,latent", [("sd21", 96), ("sd15", 64)], ids=["sd21-768px", "sd15-512px"])
def test_short_loop_within_bound(name, latent):
    """`PwWSampler` (CUDA graph, LMS, 3 steps, packed maps of every level, the KV cache and the sampler kernels) against
    the restated reference loop (two batch-1 forwards per step) run in fp32 (reference) and with the emulating oracle on
    the plain fp16 route (baseline), on the final latents."""
    dtype, steps = F16, 3
    m = models(name, dtype)
    cond, uncond = pww_dicts(m.cfg, latent * 8, dtype)
    ctx_c, ctx_u = cond["CONTEXT_TENSOR"].to(dtype), uncond["CONTEXT_TENSOR"].to(dtype)
    lat = (torch.randn(1, 4, latent, latent, generator=torch.manual_seed(0)) * _scheduler(steps).init_noise_sigma).cuda()

    with _fast_route(True):
        try:
            P.patch_unet(m.unet)
            subj = PwWSampler(m.unet, _scheduler(steps), [_with_ctx(cond, ctx_c.float())],
                              [_with_ctx(uncond, ctx_u.float())], lat, WF, 7.5, use_graph=True).run().float()
        finally:
            P.unpatch_all()
    with _fast_route(False):
        try:
            oracle_loop.patch_with_oracle(m.unet, emulate_dtype=dtype)
            base = oracle_loop.reference_denoise_loop(m.unet, _scheduler(steps), _with_ctx(cond, ctx_c),
                                                      _with_ctx(uncond, ctx_u), lat, WF).float()
        finally:
            _drop_oracle_patch()
    with _fast_route(False), _no_tf32():
        try:
            oracle_loop.patch_with_oracle(m.ref)
            ref = oracle_loop.reference_denoise_loop(m.ref, _scheduler(steps), _with_ctx(cond, ctx_c.float()),
                                                     _with_ctx(uncond, ctx_u.float()), lat, WF)
        finally:
            _drop_oracle_patch()
    assert_within_bound(f"loop {name} {latent * 8}px fp16", {"latents": subj}, {"latents": base}, {"latents": ref},
                        dtype)


# ---------------------------------------------------------------------------------------------------------------------
# 3. ControlNet residuals and adapter features at the 13 real skip shapes (sd15, 512 px, fp16)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("rows", [2, 1], ids=["both-rows", "guess-mode"])
@pytest.mark.parametrize("scaled", [False, True], ids=["plain-add", "control-scales"])
def test_controlnet_residuals_within_bound(scaled, rows):
    """12 down residuals and a mid residual at batch 2 (stacked cond + uncond contexts), for both rows or for the cond
    row only (guess mode); added plainly, or scaled per image through CONTROL_SCALES in a context dict whose weight
    function is zero (so attention stays unbiased)."""
    dtype = F16
    m = models("sd15", dtype)
    case = Case(m.cfg, 64, dtype, "scaled" if scaled else "tensor", batch=2)
    g = torch.Generator().manual_seed(11)
    shapes, mid = skip_shapes(m.cfg, 64)
    case.extra["down_block_additional_residuals"] = [_rand((rows,) + s, g, dtype, 0.5) for s in shapes]
    case.extra["mid_block_additional_residual"] = _rand((rows,) + mid, g, dtype, 0.5)
    case.control_scales = (torch.rand(len(shapes) + 1, rows, generator=g) * 1.5 + 0.25).cuda()
    subj, base, ref = run_case(m, case)
    assert_within_bound(f"controlnet {'scaled' if scaled else 'plain'} rows={rows}", subj, base, ref, dtype)


def adapter_features(cfg, latent, rows, dtype, seed=12):
    g = torch.Generator().manual_seed(seed)
    shapes, _ = skip_shapes(cfg, latent)
    last = [shapes[1 + (cfg.layers_per_block + 1) * i + cfg.layers_per_block - 1] for i in range(len(cfg.block_out_channels))]
    return [_rand((rows,) + s, g, dtype, 0.5) for s in last]


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [2, 1], ids=["both-rows", "first-row"])
def test_adapter_features_within_bound(rows):
    """Four adapter features, one per encoder level, for both rows of a batch-2 forward or for the first row only."""
    dtype = F16
    m = models("sd15", dtype)
    case = Case(m.cfg, 64, dtype, "tensor", batch=2)
    case.extra["down_intrablock_additional_residuals"] = adapter_features(m.cfg, 64, rows, dtype)
    subj, base, ref = run_case(m, case)
    assert_within_bound(f"adapter rows={rows}", subj, base, ref, dtype)


# ---------------------------------------------------------------------------------------------------------------------
# 4. peaked attention
# ---------------------------------------------------------------------------------------------------------------------
def peakedness(ref, name: str, run):
    """Mean over rows and heads of the largest softmax probability of the self-attention module `name` of `ref` during
    `run()` (its to_q / to_k outputs recorded by hooks; the oracle's patched __call__ bypasses the module's own hooks)."""
    attn = dict(ref.named_modules())[name]
    got = {}
    hs = [attn.to_q.register_forward_hook(lambda mod, a, out: got.__setitem__("q", out.detach().float())),
          attn.to_k.register_forward_hook(lambda mod, a, out: got.__setitem__("k", out.detach().float()))]
    try:
        run()
    finally:
        for h in hs:
            h.remove()
    q, k = got["q"], got["k"]
    b, n, c = q.shape
    d = c // attn.heads
    qh = q.reshape(b, n, attn.heads, d).transpose(1, 2)
    kh = k.reshape(b, k.shape[1], attn.heads, d).transpose(1, 2)
    with _no_tf32():
        p = (qh @ kh.transpose(-1, -2) * attn.scale).softmax(-1)
    return p.max(-1).values.mean().item()


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["auto", "native"])
def test_sharpened_attention_within_bound(impl):
    """sd15 at 512 px, fp16, paint-with-words dict, with every to_q weight multiplied by SHARPEN: attention at the
    1024-key level is peaked (checked on the reference), so a wrong running maximum, a lost rescale or a mis-masked tail
    would move the output."""
    dtype = F16
    _CACHE.pop("models", None)
    unet, ref = _to_device(_host("sd15"), dtype, SHARPEN)
    try:
        m = _Models("sd15-sharpened", dtype, unet, ref)
        case = Case(m.cfg, 64, dtype, "pww")
        attention.SELF_ATTN_IMPL = impl
        kw_ref = case.kw(torch.float32)
        with _fast_route(False), _no_tf32():
            try:
                oracle_loop.patch_with_oracle(ref)
                peak = peakedness(ref, "down_blocks.1.attentions.0.transformer_blocks.0.attn1", lambda: ref(**kw_ref))
            finally:
                _drop_oracle_patch()
        print(f"\n[sharpened x{SHARPEN}] mean largest softmax probability at the 1024-key level: {peak:.4f}")
        assert peak > PEAKED, peak
        subj, base, refo = run_case(m, case)
        assert_within_bound(f"sharpened x{SHARPEN} {impl}", subj, base, refo, dtype)
    finally:
        del unet, ref
        gc.collect()
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# 5. the harness can fail: one wrapper made slightly wrong at a time
# ---------------------------------------------------------------------------------------------------------------------
def _mutant_self_attention(q, k, v, heads, scale):
    """Self-attention that ignores the last 16 keys.  The native kernel takes one sequence length for queries and keys,
    so the truncated keys go through the library call."""
    B, N, C = q.shape
    D = C // heads
    n = k.shape[1] - 16
    qh = q.reshape(B, N, heads, D).transpose(1, 2)
    kh = k[:, :n].reshape(B, n, heads, D).transpose(1, 2)
    vh = v[:, :n].reshape(B, n, heads, D).transpose(1, 2)
    return F.scaled_dot_product_attention(qh, kh, vh, scale=scale).transpose(1, 2).reshape(B, N, C)


def _mutant_block_biases(block):
    """The residual epilogue's bias without the shortcut's."""
    tb, _ = _ORIG["block_biases"](block)
    return tb, block.conv2.bias.float().contiguous()


def _mutant_project_time_embeddings(self, temb):
    """Each block reads the columns after its own slice of the batched time projection (wrapping at the end)."""
    _ORIG["project_time"](self, temb)
    res = U._resnets(self)
    t_all = torch.cat([r._pww_t for r in res], 1)
    total, off = t_all.shape[1], 0
    for r in res:
        n = r._pww_t.shape[1]
        cols = torch.arange(off + n, off + 2 * n, device=t_all.device) % total
        object.__setattr__(r, "_pww_t", t_all[:, cols])
        off += n


def _mutant_down_forward(self, x, temb, ctx, adapter_feature=None):
    """The adapter feature added after the level's last skip was taken (on the fast route)."""
    if adapter_feature is None or not fused_ops.is_fast(x):
        return _ORIG["down_forward"](self, x, temb, ctx, adapter_feature)
    x, outs = _ORIG["down_forward"](self, x, temb, ctx, None)
    if self.downsamplers is None:
        return U.add_adapter_feature(x, adapter_feature), outs
    pre = outs[-2]                                   # the last layer's output, before the downsampler
    x = self.downsamplers[0](U.add_adapter_feature(pre, adapter_feature))
    return x, outs[:-1] + [x]


_ORIG = {"block_biases": U._block_biases, "project_time": U._project_time_embeddings,
         "down_forward": U._DownBlock.forward}

MUTATIONS = {
    "self-attention-drops-keys": ((attention, "self_attention", _mutant_self_attention), "down_blocks.0.attentions.0"),
    "shortcut-bias-lost": ((U, "_block_biases", _mutant_block_biases), "down_blocks.1.resnets.0"),
    "time-projection-off-by-one": ((U.UNet2DConditionModel, "_project_time_embeddings",
                                    _mutant_project_time_embeddings), "down_blocks.0.resnets.0"),
    "adapter-feature-too-late": ((U._DownBlock, "forward", _mutant_down_forward), "down_blocks.0.attentions.1"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_is_caught_where_it_enters(mutation, monkeypatch):
    """sd15 at 256 px, fp16, paint-with-words dict (plus adapter features for the adapter mutation): the comparison must
    report the mutated wrapper's module as the first one out of bound."""
    (obj, attr, fn), expected = MUTATIONS[mutation]
    dtype = F16
    m = models("sd15", dtype)
    case = Case(m.cfg, 32, dtype, "pww")
    if mutation == "adapter-feature-too-late":
        case.extra["down_intrablock_additional_residuals"] = adapter_features(m.cfg, 32, 1, dtype)
    monkeypatch.setattr(obj, attr, fn)
    subj, base, ref = run_case(m, case)
    check_reference(ref)
    rows, bad = compare(subj, base, ref, K, FLOOR[dtype])
    at = dict((r[0], r) for r in rows)[expected]
    print(f"\n[mutation {mutation}] at {expected}: subject {at[1][0]:.3e} {at[1][1]:.3e} | baseline {at[2][0]:.3e} "
          f"{at[2][1]:.3e}; first violation {bad}")
    assert bad is not None and bad[0] == expected, (mutation, bad)


# ---------------------------------------------------------------------------------------------------------------------
# 6. the comparison code itself, on the CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_compare_reports_first_perturbed_block_on_cpu():
    """Tiny UNet on the CPU: fp64 reference, fp32 subject and baseline; a hook adds 1e-2 to one ResNet block's output
    in the subject, and exactly that block is reported as the first failure."""
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0)
    ref = copy.deepcopy(unet).double()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, cfg.in_channels, cfg.sample_size, cfg.sample_size, generator=g)
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=g)
    t = torch.tensor([500.0])
    target = "down_blocks.1.resnets.1"
    h = dict(unet.named_modules())[target].register_forward_hook(lambda mod, a, out: out + 1e-2)
    try:
        subj, _ = record_outputs(unet, lambda: unet(x, t, encoder_hidden_states=ctx))
    finally:
        h.remove()
    base, _ = record_outputs(unet, lambda: unet(x, t, encoder_hidden_states=ctx))
    refo, _ = record_outputs(ref, lambda: ref(x.double(), t, encoder_hidden_states=ctx.double()), torch.float64)
    check_reference(refo)
    names = list(refo)
    assert names.index(target) < names.index("down_blocks.1") < names.index("conv_out")
    rows, bad = compare(subj, base, refo, K, FLOOR[torch.float16])
    assert bad is not None and bad[0] == target, bad
    assert all(max(es) < 1e-4 for name, es, _ in rows[:names.index(target)])
