"""The per-element bounds of `tests/unet_ops_bound.py`, checked on the CPU from both sides.

  * Loose enough: a float32 emulation of each kernel's arithmetic, in the kernel's order and rounded to E once, passes
    at every CPU-sized shape of the GPU lists, in fp16 and bf16.
  * Tight enough: plausible wrong kernels (computed in fp64, rounded to E) fail at one or more of those shapes; each
    mutation test prints the shapes that caught it.

The emulations sum in fp32 chains shaped like the kernels' but not in their exact order, so they show the
bound's margin over a correct kernel's roundings, not the kernels' exact bits; the GPU file runs the kernels.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import unet_ops_bound as U

CPU_ELEMS = 3 << 20          # the CPU cases: GPU-list shapes up to this many activation elements
EPS = 1e-5


# ---- the checker itself ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", U.DTYPES, ids=U.DTYPE_IDS)
def test_ulp_is_the_spacing_of_E(dtype):
    r = torch.tensor([1.0, 1.5, 2.0, 3.9, 1e-3, -100.0, 0.0], dtype=torch.float64)
    p = 10 if dtype == torch.float16 else 7
    want = [2.0 ** -p, 2.0 ** -p, 2.0 ** (1 - p), 2.0 ** (1 - p), 2.0 ** (-10 - p), 2.0 ** (6 - p),
            2.0 ** ((-14 if dtype == torch.float16 else -126) - p)]
    assert U.ulp_E(r, dtype).tolist() == want
    # E's next value away from zero is exactly one ulp_E away (normal range)
    e = r[:6].to(dtype)
    nxt = (e.view(torch.int16) + 1).view(dtype)
    assert ((nxt.double() - e.double()).abs() == U.ulp_E(e.double(), dtype)).all()


def test_checker_passes_one_ulp_and_names_the_worst_element():
    ref = torch.full((2, 3, 8), 1.0, dtype=torch.float64)
    terms = torch.zeros_like(ref)
    got = ref.clone().half()
    got[1, 2, 5] = 1.0 + 2.0 ** -10                                   # one ulp: inside
    assert U.check_within(got, ref, terms, torch.float16, U.K_GN) == 1.0
    got[0, 1, 3] = 1.0 + 2.0 ** -9                                    # two ulps: outside
    got[1, 0, 7] = 1.0 + 3 * 2.0 ** -10                               # three: the worst
    with pytest.raises(AssertionError, match=r"2 of 48 elements.*image 1, row 0, channel 7"):
        U.check_within(got, ref, terms, torch.float16, U.K_GN)
    got = ref.clone().half()
    got[0, 0, 0] = math.nan
    with pytest.raises(AssertionError, match="image 0, row 0, channel 0"):
        U.check_within(got, ref, terms, torch.float16, U.K_GN)
    # the fp32 term widens the allowance per element
    got = ref.clone().half()
    got[0, 0, 1] = 1.0 + 2.0 ** -9
    terms[0, 0, 1] = 2.0 ** -10 / U.K_GN
    U.check_within(got, ref, terms, torch.float16, U.K_GN)


def test_checker_accepts_inf_only_where_the_reference_overflows():
    ref = torch.tensor([[7e4, -9e4, 6e4, 65519.0]], dtype=torch.float64)
    terms = torch.zeros_like(ref)
    got = torch.tensor([[math.inf, -math.inf, 6e4, 65504.0]]).half()
    U.check_within(got, ref, terms, torch.float16, U.K_GEGLU)
    with pytest.raises(AssertionError, match="channel 2"):
        U.check_within(torch.tensor([[math.inf, -math.inf, math.inf, 65504.0]]).half(), ref, terms, torch.float16,
                       U.K_GEGLU)
    with pytest.raises(AssertionError, match="channel 0"):
        U.check_within(torch.tensor([[-math.inf, -math.inf, 6e4, 65504.0]]).half(), ref, terms, torch.float16,
                       U.K_GEGLU)


# ---- GroupNorm -------------------------------------------------------------------------------------------------------
def _chained_sum(t, G):
    """[B, G] fp32 sums of t [B, HW, C] over each group's rows and channels, in fp32 chains like the kernel's: each
    channel's rows summed in order within row chunks (at most 64 chunks, as gn_split makes), then the chunks and the
    group's channels."""
    B, HW, C = t.shape
    chunks = min(64, HW)
    rpc = -(-HW // chunks)
    t = torch.cat([t, t.new_zeros(B, chunks * rpc - HW, C)], 1).reshape(B, chunks, rpc, C)
    part = t[:, :, 0]
    for r in range(1, rpc):
        part = part + t[:, :, r]
    return part.sum(1).reshape(B, G, C // G).sum(-1)


def gn_emulate(x, gamma, beta, G, eps, add=None, silu=False):
    """gn_stats_kernel + gn_apply_kernel in float32: sums of d = x + (add - shift) about the group's first element,
    var = E[d^2] - E[d]^2, sc = rstd * gamma, sh = beta + ((add - shift) - E[d]) * sc, y = fma(x, sc, sh),
    SiLU y / (1 + exp(-y)); rounded to E."""
    B, HW, C = x.shape
    cg = C // G
    xf = x.float()
    af = add.float() if add is not None else torch.zeros(B, C)
    shift = xf[:, 0, ::cg] + af[:, ::cg]                                       # [B, G]
    d = xf + (af - shift.repeat_interleave(cg, 1))[:, None, :]
    n = float(HW * cg)
    dm = _chained_sum(d, G) / n
    var = (_chained_sum(d * d, G) / n - dm * dm).clamp_min(0.0)
    rstd = torch.rsqrt(var + eps)
    sc = rstd.repeat_interleave(cg, 1) * gamma.float()
    sh = beta.float() + ((af - shift.repeat_interleave(cg, 1)) - dm.repeat_interleave(cg, 1)) * sc
    y = (xf.double() * sc.double()[:, None, :] + sh.double()[:, None, :]).float()    # fma: one rounding
    if silu:
        y = y / (1.0 + torch.exp(-y))
    return y.to(x.dtype)


def gn_mutant(kind, x, gamma, beta, G, eps, add=None, silu=False):
    """A wrong GroupNorm, in fp64, rounded to E."""
    B, HW, C = x.shape
    cg = C // G
    xd = x.double() + (add.double()[:, None, :] if add is not None else 0.0)
    grp = xd.reshape(B, HW, G, cg)
    mean = grp.mean(dim=(1, 3), keepdim=True)
    var = (grp - mean).pow(2).mean(dim=(1, 3), keepdim=True)
    n = HW * cg
    if kind == "unbiased_var":
        var = var * n / (n - 1)
    if kind in ("mean_rounded_to_E", "mean_rounded_to_fp32"):
        mean = mean.to(x.dtype if kind == "mean_rounded_to_E" else torch.float32).double()
    rstd = 1.0 / (var.sqrt() + eps) if kind == "eps_outside_sqrt" else (var + eps).rsqrt()
    y = ((grp - mean) * rstd).reshape(B, HW, C) * gamma.double() + beta.double()
    if silu:
        s = torch.sigmoid(y)
        y = y * (s.to(x.dtype).double() if kind == "sigmoid_rounded_to_E" else s)
    return y.to(x.dtype)


def _gn_cases():
    """(id, HW, C, G, B, variant, input kind): the GPU list's CPU-sized shapes, and the extreme inputs."""
    cases = []
    for HW, C, G, B in U.GN_SHAPES:
        if B * HW * C <= CPU_ELEMS:
            for (silu, with_add), vid in zip(U.GN_VARIANTS, U.GN_VARIANT_IDS):
                cases.append((f"{HW}x{C}g{G}b{B}-{vid}", HW, C, G, B, silu, with_add, "randn"))
    for HW, C in [(4096, 320), (1024, 640)]:
        cases.append((f"{HW}x{C}-mean50", HW, C, 32, 2, False, True, "mean50"))
    cases.append(("1024x640-mean1000", 1024, 640, 32, 2, False, True, "mean1000"))      # fp16 only
    for kind in ("const", "std1e-4"):
        for HW, C, G, B in [(1024, 640, 32, 2), (33, 64, 64, 1)]:     # 64 groups of one channel: add constant per group
            for (silu, with_add), vid in zip(U.GN_VARIANTS, U.GN_VARIANT_IDS):
                cases.append((f"{HW}x{C}g{G}-{kind}-{vid}", HW, C, G, B, silu, with_add, kind))
    return cases


GN_CASES = _gn_cases()


def _gn_ids(cases):
    return [c[0] for c in cases]


@pytest.mark.parametrize("dtype", U.DTYPES, ids=U.DTYPE_IDS)
@pytest.mark.parametrize("case", GN_CASES, ids=_gn_ids(GN_CASES))
def test_groupnorm_emulation_passes(case, dtype):
    name, HW, C, G, B, silu, with_add, kind = case
    if kind == "mean1000" and dtype == torch.bfloat16:
        pytest.skip("bf16 spaces values near 1000 by 8: no variance left to normalise")
    x, gamma, beta, add = U.gn_case_inputs(HW, C, G, B, dtype, with_add, kind, seed=HW + C + B)
    ref, terms = U.gn_reference(x, gamma, beta, G, EPS, add, silu)
    worst = U.check_within(gn_emulate(x, gamma, beta, G, EPS, add, silu), ref, terms, dtype, U.K_GN, name)
    print(f"BOUND gn-emulation {name} {dtype} worst {worst:.3f} of the allowance")


def test_groupnorm_constant_case_has_constant_groups():
    x, gamma, beta, add = U.gn_case_inputs(1024, 640, 32, 2, torch.float16, True, "const", seed=1)
    xin = (x.float() + add.float()[:, None, :]).reshape(2, 1024, 32, 20)
    spread = xin.amax(dim=(1, 3)) - xin.amin(dim=(1, 3))
    assert (spread[:, 0::2] == 0).all() and (spread[:, 1::2] > 0).all()


GN_MUTATIONS = [
    # (mutation, cases that may show it: an empty filter means every case)
    ("unbiased_var", lambda c: c[7] == "randn"),
    ("mean_rounded_to_E", lambda c: c[7] == "mean50"),
    # the apply kernel's earlier sh = beta + (add - fp32(shift + E[d])) * sc: shows where |add| >> std
    ("mean_rounded_to_fp32", lambda c: c[7] == "std1e-4" and c[6]),
    ("sigmoid_rounded_to_E", lambda c: c[5]),
    ("eps_outside_sqrt", lambda c: c[7] in ("std1e-4", "const")),
]


@pytest.mark.parametrize("dtype", U.DTYPES, ids=U.DTYPE_IDS)
@pytest.mark.parametrize("kind,applies", GN_MUTATIONS, ids=[m[0] for m in GN_MUTATIONS])
def test_groupnorm_mutation_fails(kind, applies, dtype):
    caught = []
    for case in filter(applies, GN_CASES):
        name, HW, C, G, B, silu, with_add, ikind = case
        x, gamma, beta, add = U.gn_case_inputs(HW, C, G, B, dtype, with_add, ikind, seed=HW + C + B)
        ref, terms = U.gn_reference(x, gamma, beta, G, EPS, add, silu)
        try:
            U.check_within(gn_mutant(kind, x, gamma, beta, G, EPS, add, silu), ref, terms, dtype, U.K_GN, name)
        except AssertionError:
            caught.append(name)
    print(f"BOUND gn mutation {kind} {dtype} caught by {caught}")
    assert caught, f"{kind} passes the bound at every shape"


# ---- GEGLU -----------------------------------------------------------------------------------------------------------
def geglu_emulate(h):
    """geglu_kernel in float32: a * (0.5 g (1 + erf(g / sqrt 2))), rounded to E."""
    I = h.shape[-1] // 2
    a, g = h[:, :I].float(), h[:, I:].float()
    return (a * (0.5 * g * (1.0 + torch.erf(g * 0.70710678118654752)))).to(h.dtype)


def geglu_mutant(kind, h):
    I = h.shape[-1] // 2
    a, g = h[:, :I].double(), h[:, I:].double()
    if kind == "tanh_gelu":
        return (a * F.gelu(g, approximate="tanh")).to(h.dtype)
    return (a * F.gelu(g).to(h.dtype).double()).to(h.dtype)      # "gelu_rounded_to_E"


GEGLU_CASES = [(M, I) for M in U.GEGLU_M for I in U.GEGLU_I if M * I <= CPU_ELEMS]


@pytest.mark.parametrize("dtype", U.DTYPES, ids=U.DTYPE_IDS)
@pytest.mark.parametrize("M,I", GEGLU_CASES)
def test_geglu_emulation_passes(M, I, dtype):
    h = U.geglu_inputs(M, I, dtype, seed=M + I)
    ref, terms = U.geglu_reference(h)
    worst = U.check_within(geglu_emulate(h), ref, terms, dtype, U.K_GEGLU, f"geglu {M}x{I}")
    print(f"BOUND geglu-emulation {M}x{I} {dtype} worst {worst:.3f} of the allowance")


def test_geglu_cancellation_is_the_formulas():
    """Below g ~ -4, 1 + erf(g / sqrt 2) cancels in fp32: 4 % off at g = -5 and exactly 0 from g = -6 on, while the
    fp64 GELU is -1.4e-6 and -6e-9 there.  torch's fp32 F.gelu has the same formula and the same zeros, which the
    fast route has to match; the bound's |a| |g| term carries it."""
    g = torch.tensor([-5.0, -6.0, -8.0, -10.0])
    emu = 0.5 * g * (1.0 + torch.erf(g * 0.70710678118654752))
    exact = 0.5 * g.double() * torch.special.erfc(-g.double() / math.sqrt(2.0))
    assert abs(float(emu[0]) / float(exact[0]) - 1.0) > 0.01
    assert (emu[1:] == 0).all() and (F.gelu(g)[1:] == 0).all() and (exact[1:] != 0).all()
    assert ((emu.double() - exact).abs() <= 1.3 * 2.0 ** -24 * g.double().abs()).all()


def test_geglu_overflow_is_inf_like_torch():
    h = torch.tensor([[300.0, -300.0, 2.0, 300.0, 300.0, 3.0]]).half()        # a | g, I = 3
    got = geglu_emulate(h)
    ref, terms = U.geglu_reference(h)
    assert got[0, 0] == math.inf and got[0, 1] == -math.inf
    assert torch.equal(got[0, :2], (h[:, :3] * F.gelu(h[:, 3:].float()).half())[0, :2])
    U.check_within(got, ref, terms, torch.float16, U.K_GEGLU, "geglu overflow")


GEGLU_MUTATIONS = ["tanh_gelu", "gelu_rounded_to_E"]


@pytest.mark.parametrize("dtype", U.DTYPES, ids=U.DTYPE_IDS)
@pytest.mark.parametrize("kind", GEGLU_MUTATIONS)
def test_geglu_mutation_fails(kind, dtype):
    caught = []
    for M, I in GEGLU_CASES:
        h = U.geglu_inputs(M, I, dtype, seed=M + I)
        ref, terms = U.geglu_reference(h)
        try:
            U.check_within(geglu_mutant(kind, h), ref, terms, dtype, U.K_GEGLU, f"{M}x{I}")
        except AssertionError:
            caught.append(f"{M}x{I}")
    print(f"BOUND geglu mutation {kind} {dtype} caught by {caught}")
    assert caught, f"{kind} passes the bound at every shape"


# ---- add + LayerNorm -------------------------------------------------------------------------------------------------
def ln_emulate(x, res, gamma, beta, eps):
    """add_layernorm_kernel in float32: s = E(x + res), mean, sum of (s - mean)^2, rsqrt, (s - mean) * rstd * gamma +
    beta; (s, y) in E."""
    s = (x.float() + res.float()).to(x.dtype) if res is not None else x
    v = s.float()
    C = v.shape[-1]
    mean = v.sum(-1, keepdim=True) / C
    d = v - mean
    rstd = torch.rsqrt((d * d).sum(-1, keepdim=True) / C + eps)
    return s, (d * rstd * gamma.float() + beta.float()).to(x.dtype)


def ln_mutant(kind, s, gamma, beta, eps):
    sd = s.double()
    C = sd.shape[-1]
    mu = sd.mean(-1, keepdim=True)
    var = (sd - mu).pow(2).mean(-1, keepdim=True)
    if kind == "unbiased_var":
        var = var * C / (C - 1)
    rstd = 1.0 / (var.sqrt() + eps) if kind == "eps_outside_sqrt" else (var + eps).rsqrt()
    n = (sd - mu) * rstd
    if kind == "normalised_rounded_to_E":
        n = n.to(s.dtype).double()
    return (n * gamma.double() + beta.double()).to(s.dtype)


# (M, C, mean, std of x): the GPU list's C at CPU-sized M, a residual stream of mean 100, fp16 magnitudes near 2000,
# and rows of std 1e-3 (below sqrt(eps) ~ 3e-3: eps sets rstd)
LN_CASES = ([(M, C, 0.0, 2.0) for C in U.LN_C for M in (1, 7, 8, 256)]
            + [(64, C, 100.0, 1.0) for C in (320, 1280, 2048)] + [(64, 1280, 2000.0, 20.0), (64, 1280, 0.0, 1e-3)])


def _ln_id(c):
    return f"{c[0]}x{c[1]}-mean{c[2]:g}-std{c[3]:g}"


@pytest.mark.parametrize("dtype", U.DTYPES, ids=U.DTYPE_IDS)
@pytest.mark.parametrize("with_res", [True, False], ids=["res", "nores"])
@pytest.mark.parametrize("case", LN_CASES, ids=[_ln_id(c) for c in LN_CASES])
def test_layernorm_emulation_passes(case, with_res, dtype):
    M, C, mean, std = case
    x, res, gamma, beta = U.ln_inputs(M, C, dtype, seed=M + C, mean=mean, std=std)
    s, y = ln_emulate(x, res if with_res else None, gamma, beta, EPS)
    ref, terms = U.ln_reference(s, gamma, beta, EPS)
    worst = U.check_within(y, ref, terms, dtype, U.K_LN, _ln_id(case))
    print(f"BOUND ln-emulation {_ln_id(case)} {dtype} worst {worst:.3f} of the allowance")


LN_MUTATIONS = ["unbiased_var", "normalised_rounded_to_E", "eps_outside_sqrt"]


@pytest.mark.parametrize("dtype", U.DTYPES, ids=U.DTYPE_IDS)
@pytest.mark.parametrize("kind", LN_MUTATIONS)
def test_layernorm_mutation_fails(kind, dtype):
    caught = []
    for case in LN_CASES:
        M, C, mean, std = case
        x, res, gamma, beta = U.ln_inputs(M, C, dtype, seed=M + C, mean=mean, std=std)
        s = (x.float() + res.float()).to(dtype)
        ref, terms = U.ln_reference(s, gamma, beta, EPS)
        try:
            U.check_within(ln_mutant(kind, s, gamma, beta, EPS), ref, terms, dtype, U.K_LN, _ln_id(case))
        except AssertionError:
            caught.append(_ln_id(case))
    print(f"BOUND ln mutation {kind} {dtype} caught by {caught}")
    assert caught, f"{kind} passes the bound at every shape"
