"""GPU parity of the CUDA path (through the C ABI) against the oracle on identical seeded inputs.

Tolerances (SURVEY.md 8c, frozen here):
  * statistic scalar: relative 2^-10 (one fp16 ulp) against the oracle's fp16-emulating form;
  * attention output vs the fp32 oracle:            max|d| <= 2e-3 * max|out|  (fp16 storage of Q/K/V/P/O);
  * attention output vs the fp16-emulating oracle:  max|d| <= 1.5e-3 * max|out|  (the kernel keeps S and the softmax
    in fp32 and normalises O instead of P, so it sits between the two oracles; the oracles themselves differ by
    up to ~8e-4 * max|out| on these inputs).
"""
import math

import numpy as np
import pytest
import torch

from oracle import pww_oracle as O
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import attention as A

pytestmark = pytest.mark.gpu

SD15_512 = [(4096, 8, 40), (1024, 8, 80), (256, 8, 160), (64, 8, 160)]
SD15_256 = [(16, 8, 160)]
SD21_768 = [(9216, 5, 64), (2304, 10, 64), (576, 20, 64), (144, 20, 64)]
RAGGED = [(100, 8, 40), (1, 2, 64), (129, 3, 80), (333, 1, 160)]


def _inputs(B, N, H, D, T, seed):
    g = torch.Generator().manual_seed(seed)
    C = H * D
    q = (torch.randn(B, N, C, generator=g) * 0.5).half()
    k = (torch.randn(B, T, C, generator=g) * 0.5).half()
    v = (torch.randn(B, T, C, generator=g) * 0.5).half()
    w = torch.zeros(B, N, T)
    for b in range(B):                      # sparse columns like the real maps, plus overlap
        cols = torch.randperm(T, generator=g)[:9]
        for c in cols:
            w[b, :, c] += (torch.rand(N, generator=g) > 0.6).float() * float(torch.rand(1, generator=g) * 2)
    return q, k, v, w


def _oracle(q, k, v, H, scale, w, g, stat, emulate):
    outs, stats = [], []
    for b in range(q.shape[0]):
        box = {}

        def bias_fn(s, b=b):
            m = s.max() if stat == "max" else s.std()
            box["m"] = float(m)
            return g * w[b] * m.float() if w is not None else 0.0
        outs.append(O.attention_core(q[b:b + 1].float(), k[b:b + 1].float(), v[b:b + 1].float(), H, scale,
                                     bias_fn if w is not None else None, emulate_fp16=emulate))
        stats.append(box.get("m", 0.0))
    return torch.cat(outs, 0), stats


IMPLS = ["fused", "dense"]      # one-launch kernel on packed maps | round-1 pair of launches on the dense fp32 map


def _run(q, k, v, H, scale, w, g, stat, idx=None, impl="fused"):
    dev = "cuda"
    gs = torch.tensor([g], dtype=torch.float32, device=dev)
    old = A.XATTN_IMPL
    A.XATTN_IMPL = impl
    try:
        out, st = A.cross_attention(q.to(dev), k.to(dev), v.to(dev), H, scale,
                                    None if w is None else w.to(dev), None if idx is None else idx.to(dev),
                                    _native.PWW_STAT_MAX if stat == "max" else _native.PWW_STAT_STD, gs,
                                    return_stats=True)
        torch.cuda.synchronize()
    finally:
        A.XATTN_IMPL = old
    return out.float().cpu(), (None if st is None else st.cpu())


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D", SD15_512 + SD15_256 + SD21_768 + RAGGED)
@pytest.mark.parametrize("stat", ["max", "std"])
def test_bias_path_matches_oracle(N, H, D, stat, impl):
    if stat == "std" and N * H > 40000:
        pytest.skip("std covered at the smaller sizes; max covers the large ones")
    T, B = 77, 1
    q, k, v, w = _inputs(B, N, H, D, T, seed=N * 131 + D)
    scale = D ** -0.5
    g = 0.4 * math.log(1 + 7.0) if stat == "max" else 0.5 * math.log(1 + 7.0 ** 2)
    got, st = _run(q, k, v, H, scale, w, g, stat, impl=impl)
    ref16, st16 = _oracle(q, k, v, H, scale, w, g, stat, emulate=True)
    ref32, _ = _oracle(q, k, v, H, scale, w, g, stat, emulate=False)
    if N * H * T > 1:
        assert abs(float(st[0]) - st16[0]) <= 2 ** -10 * abs(st16[0]) + 1e-6, (float(st[0]), st16[0])
    amax = ref32.abs().max().item()
    assert (got - ref16).abs().max().item() <= 1.5e-3 * amax
    assert (got - ref32).abs().max().item() <= 2e-3 * amax


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D", [(4096, 8, 40), (64, 8, 160), (576, 20, 64), (1024, 8, 80)])
def test_plain_cross_attention_matches_oracle(N, H, D, impl):
    """Tensor context / uncond dict: no bias (paint_with_words.py:107-110)."""
    q, k, v, _ = _inputs(2, N, H, D, 77, seed=7)
    got, st = _run(q, k, v, H, D ** -0.5, None, 0.0, "max", impl=impl)
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, None, 0.0, "max", emulate=False)
    assert st is None
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("T", [1, 16, 41, 77, 80])
def test_key_lengths(T, impl):
    N, H, D = 256, 8, 40
    q, k, v, w = _inputs(1, N, H, D, T, seed=T)
    g = 0.7
    got, st = _run(q, k, v, H, D ** -0.5, w, g, "max", impl=impl)
    ref32, st32 = _oracle(q, k, v, H, D ** -0.5, w, g, "max", emulate=False)
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


@pytest.mark.parametrize("impl", IMPLS)
def test_batched_cfg_semantics_per_image_stats(impl):
    """[cond0, uncond, cond1] in one call: per-image statistic, index -1 = no bias, maps picked by index."""
    N, H, D, T = 1024, 8, 80, 77
    q, k, v, w = _inputs(3, N, H, D, T, seed=99)
    q[2] *= 3.0                                     # make the images' maxima very different
    idx = torch.tensor([1, -1, 0], dtype=torch.int32)
    g = 0.4 * math.log(1 + 3.0)
    got, st = _run(q, k, v, H, D ** -0.5, w[:2].contiguous(), g, "max", idx, impl=impl)
    w_eff = torch.stack([w[1], torch.zeros_like(w[0]), w[0]])
    ref, stats = _oracle(q, k, v, H, D ** -0.5, w_eff, g, "max", emulate=False)
    ref_plain, _ = _oracle(q[1:2], k[1:2], v[1:2], H, D ** -0.5, None, 0.0, "max", emulate=False)
    amax = ref.abs().max().item()
    assert (got[0] - ref[0]).abs().max().item() <= 2e-3 * amax
    assert (got[2] - ref[2]).abs().max().item() <= 2e-3 * amax
    assert (got[1] - ref_plain[0]).abs().max().item() <= 2e-3 * amax
    assert float(st[1]) == 0.0 and abs(float(st[2]) - stats[2]) <= 2e-3 * abs(stats[2])
    # batching does not change an image's result (sharding invariance): bit-identical
    solo, _ = _run(q[2:3], k[2:3], v[2:3], H, D ** -0.5, w[0:1].contiguous(), g, "max", impl=impl)
    assert torch.equal(solo[0], got[2])


def test_strided_views_no_copy_semantics():
    """q/k/v as column slices of one fused [B,L,3C] projection buffer (row stride 3C)."""
    N, H, D, T = 256, 8, 40, 77
    C = H * D
    q, k, v, w = _inputs(1, N, H, D, T, seed=5)
    kv = torch.cat([k, v], -1).cuda()               # [1,T,2C]
    out = A.cross_attention(q.cuda(), kv[..., :C], kv[..., C:], H, D ** -0.5)
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, None, 0.0, "max", emulate=False)
    assert (out.float().cpu() - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


@pytest.mark.parametrize("impl", IMPLS)
def test_stats_workspace_is_self_cleaning(impl):
    N, H, D = 1024, 8, 80
    q, k, v, w = _inputs(2, N, H, D, 77, seed=3)
    a, sa = _run(q, k, v, H, D ** -0.5, w, 0.5, "std", impl=impl)
    b, sb = _run(q, k, v, H, D ** -0.5, w, 0.5, "std", impl=impl)
    assert torch.equal(a, b) and torch.equal(sa, sb)          # deterministic, counters reset


def test_unsupported_shape_raises():
    q = torch.zeros(1, 64, 96, dtype=torch.float16, device="cuda")
    kv = torch.zeros(1, 77, 96, dtype=torch.float16, device="cuda")
    with pytest.raises(_native.NativeError):
        A.cross_attention(q, kv, kv, 2, 0.1)                  # D=48: no kernel, no fallback
    for T in (81, 128, 200):                                  # only Stable Diffusion's key lengths (<= 80) have a kernel
        kv = torch.zeros(1, T, 80, dtype=torch.float16, device="cuda")
        with pytest.raises(_native.NativeError):
            A.cross_attention(torch.zeros(1, 64, 80, dtype=torch.float16, device="cuda"), kv, kv, 2, 0.1)


@pytest.mark.parametrize("impl", IMPLS)
def test_real_weight_map_aurora(golden, impl):
    """aurora_1 map at N=4096 (config 2 of BASELINE.json), default-style weight function."""
    mb = golden["mask_builder"]
    w = torch.from_numpy(mb["aurora_512_w8"])[None]
    q, k, v, _ = _inputs(1, 4096, 8, 40, 77, seed=2026)
    g = 0.4 * math.log(1 + 14.6146)
    got, st = _run(q, k, v, 8, 40 ** -0.5, w, g, "max", impl=impl)
    ref32, stats = _oracle(q, k, v, 8, 40 ** -0.5, w, g, "max", emulate=False)
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("B", [1, 2])
def test_mask_barrier_stress_cold_maps(B, impl):
    """Round 1's intermittent failure (VERDICT r01): with > 1 mask group per CTA a softmax group could read the shared
    mask tile before it had landed.  Run the failing launch shapes (N=4096, H=8, D=40; B=1 and the bench's B=2 with one
    biased image) 200 times, each time with a weight map that is cold in L2 (fresh copy + an L2-sized write in
    between), and require every output to be bit-identical to the first one, which is checked against the oracle."""
    N, H, D, T = 4096, 8, 40, 77
    q, k, v, w = _inputs(B, N, H, D, T, seed=4242 + B)
    g = 0.4 * math.log(1 + 7.0)
    idx = torch.tensor([0] + [-1] * (B - 1), dtype=torch.int32)
    w1 = w[:1].contiguous()
    w_eff = torch.cat([w1, torch.zeros(B - 1, N, T)], 0)
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, w_eff, g, "max", emulate=False)
    dev = "cuda"
    qd, kd, vd, idxd = q.to(dev), k.to(dev), v.to(dev), idx.to(dev)
    gs = torch.tensor([g], dtype=torch.float32, device=dev)
    flush = torch.empty(192 << 20, dtype=torch.uint8, device=dev)
    pool = [w1.to(dev).clone() for _ in range(8)]
    first = None
    bad = torch.zeros((), dtype=torch.int32, device=dev)
    A.XATTN_IMPL = impl
    packed_pool = None
    if impl == "fused":
        from paint_with_words_sd_b200.conditioning import pack_weight_map
        packed_pool = [pack_weight_map(p_) for p_ in pool]
    for i in range(200):
        wd = pool[i % 8].clone()                     # fresh allocation, never touched by a kernel before
        pk = None
        if packed_pool is not None:
            pk = (packed_pool[i % 8][0].clone(), packed_pool[i % 8][1].clone())
        flush.fill_(i & 0xFF)                        # evict Q/K/V and the maps from L2
        out = A.cross_attention(qd, kd, vd, H, D ** -0.5, wd, idxd, _native.PWW_STAT_MAX, gs, packed=pk)
        if first is None:
            first = out.clone()
        else:
            bad += (out != first).any().to(torch.int32)
    torch.cuda.synchronize()
    A.XATTN_IMPL = "auto"
    assert int(bad) == 0, f"{int(bad)} of 199 repeat launches differ from the first"
    amax = ref32.abs().max().item()
    assert (first.float().cpu() - ref32).abs().max().item() <= 2e-3 * amax


# ------------------------------------------------------------------------------------------------------------------
# one-launch kernel specifics
# ------------------------------------------------------------------------------------------------------------------
def _set_fused_grid(n):
    import ctypes
    L = _native.lib()
    L.pww_debug_set_fused_grid.argtypes = [ctypes.c_int]
    assert L.pww_debug_set_fused_grid(n) == 0


@pytest.mark.parametrize("N,H,D,B,grid", [(1024, 8, 40, 4, 8), (1024, 8, 40, 2, 3), (2304, 10, 64, 4, 16),
                                          (1024, 8, 80, 6, 12), (256, 8, 160, 8, 5), (333, 3, 40, 5, 4)])
@pytest.mark.parametrize("stat", ["max", "std"])
def test_fused_long_job_lists(N, H, D, B, grid, stat):
    """A capped persistent grid puts 10-40 jobs on every CTA: ring stages, score slots, output accumulators, the
    B-operand tile of the bias and the exchange buffers are all reused many times, and CTAs span several images."""
    T = 77
    q, k, v, w = _inputs(B, N, H, D, T, seed=B * 1000 + N + D)
    nb = (B + 1) // 2
    idx = torch.tensor([(i // 2 if i % 2 == 0 else -1) for i in range(B)], dtype=torch.int32)   # cond/uncond interleaved
    g = 0.4 * math.log(1 + 5.0)
    w_eff = torch.stack([w[i // 2] if i % 2 == 0 else torch.zeros(N, T) for i in range(B)])
    _set_fused_grid(grid)
    try:
        got, st = _run(q, k, v, H, D ** -0.5, w[:nb].contiguous(), g, stat, idx)
    finally:
        _set_fused_grid(0)
    ref32, stats = _oracle(q, k, v, H, D ** -0.5, w_eff, g, stat, emulate=False)
    amax = ref32.abs().max().item()
    assert (got - ref32).abs().max().item() <= 2e-3 * amax
    for b in range(B):
        if idx[b] < 0:
            assert float(st[b]) == 0.0
        else:
            assert abs(float(st[b]) - stats[b]) <= 2e-3 * abs(stats[b]) + 1e-6
    # the full grid gives bit-identical results: the statistic does not depend on how units are split over CTAs
    full, st_full = _run(q, k, v, H, D ** -0.5, w[:nb].contiguous(), g, stat, idx)
    if stat == "max":
        assert torch.equal(full, got) and torch.equal(st_full, st)


def test_fused_std_long_job_lists_repeat_bit_identically():
    """Long job lists with the std statistic at head dim 40: every CTA reuses its two operand stages many times and spans
    several images.  A stage overwritten while it is still being read would make the output depend on timing, so 40
    launches of that configuration must agree bit for bit (fixed grid: the std partials are summed in CTA order) and with
    the oracle."""
    N, H, D, T, B = 1024, 8, 40, 77, 4
    q, k, v, w = _inputs(B, N, H, D, T, seed=4242)
    idx = torch.tensor([0, -1, 1, -1], dtype=torch.int32)
    g = 0.4 * math.log(1 + 5.0)
    w_eff = torch.stack([w[0], torch.zeros(N, T), w[1], torch.zeros(N, T)])
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, w_eff, g, "std", emulate=False)
    _set_fused_grid(6)
    try:
        first, st0 = _run(q, k, v, H, D ** -0.5, w[:2].contiguous(), g, "std", idx)
        assert (first - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()
        for _ in range(39):
            again, st = _run(q, k, v, H, D ** -0.5, w[:2].contiguous(), g, "std", idx)
            assert torch.equal(again, first) and torch.equal(st, st0)
    finally:
        _set_fused_grid(0)


def test_fused_all_biased_and_all_unbiased_batches():
    """Batches without a partner image of the other kind (solo groups of the unit order)."""
    N, H, D, T = 1024, 8, 40, 77
    q, k, v, w = _inputs(3, N, H, D, T, seed=77)
    g = 0.9
    got, st = _run(q, k, v, H, D ** -0.5, w, g, "max")                       # all biased, identity map index
    ref32, stats = _oracle(q, k, v, H, D ** -0.5, w, g, "max", emulate=False)
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()
    idx = torch.tensor([2, -1, -1], dtype=torch.int32)                       # one biased, two unbiased
    got, st = _run(q, k, v, H, D ** -0.5, w, g, "max", idx)
    w_eff = torch.stack([w[2], torch.zeros(N, T), torch.zeros(N, T)])
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, w_eff, g, "max", emulate=False)
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


def test_default_dispatch_per_head_dim():
    """The shim's default is the one-launch kernel at every head dim."""
    for (N, H, D, launches) in ((1024, 8, 40, 1), (256, 8, 80, 1), (64, 8, 160, 1), (256, 5, 64, 1)):
        q, k, v, w = _inputs(1, N, H, D, 77, seed=N + D)
        before = _native.launch_count
        got, st = _run(q, k, v, H, D ** -0.5, w, 0.6, "max", impl="auto")
        assert _native.launch_count - before == launches
        ref32, _ = _oracle(q, k, v, H, D ** -0.5, w, 0.6, "max", emulate=False)
        assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


def test_fused_more_than_ten_columns_takes_the_dense_pair():
    """A map with 30 distinct columns cannot be packed: the shim must route it to the dense two-launch path."""
    N, H, D, T = 256, 8, 40, 77
    q, k, v, _ = _inputs(1, N, H, D, T, seed=11)
    gen = torch.Generator().manual_seed(5)
    w = torch.zeros(1, N, T)
    w[0, :, :30] = torch.rand(N, 30, generator=gen)
    from paint_with_words_sd_b200.conditioning import pack_weight_map
    assert pack_weight_map(w) is None
    before = _native.launch_count
    got, st = _run(q, k, v, H, D ** -0.5, w, 0.6, "max")
    assert _native.launch_count - before == 2
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, w, 0.6, "max", emulate=False)
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


def test_fused_is_one_launch_and_large_bias_precision():
    """One native launch per call; and the hi/lo split of map and coefficient keeps a LARGE bias exact: strength 8 with
    g = 3 puts logits at several hundred, where a plain fp16 product (2^-11 relative) would be off by ~0.1."""
    N, H, D, T = 1024, 8, 40, 77
    q, k, v, _ = _inputs(1, N, H, D, T, seed=21)
    gen = torch.Generator().manual_seed(9)
    w = torch.zeros(1, N, T)
    base = torch.rand(N, 3, generator=gen) * 8.0
    w[0, :, 4] = base[:, 0]; w[0, :, 5] = base[:, 0]; w[0, :, 20] = base[:, 1]; w[0, :, 33] = base[:, 2]
    w[0, :, 20] += base[:, 0]                                   # a token shared by two regions: its own dictionary entry
    before = _native.launch_count
    got, st = _run(q, k, v, H, D ** -0.5, w, 3.0, "max")
    assert _native.launch_count - before == 1
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, w, 3.0, "max", emulate=False)
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


def test_pack_cache_is_not_fooled_by_address_reuse():
    """The shim caches the packed form of a dense map by storage address + version; a freed map's address is routinely
    handed to the next map of the same shape by the caching allocator, so the cache must pin what it indexes."""
    N, H, D, T = 1024, 8, 40, 77
    q, k, v, w = _inputs(1, N, H, D, T, seed=31)
    g = 0.8
    a, _ = _run(q, k, v, H, D ** -0.5, w, g, "max")                   # w.to("cuda") is freed when _run returns
    w2 = torch.roll(w, 7, dims=2).contiguous()                        # same shape, different columns
    b, _ = _run(q, k, v, H, D ** -0.5, w2, g, "max")
    ref_a, _ = _oracle(q, k, v, H, D ** -0.5, w, g, "max", emulate=False)
    ref_b, _ = _oracle(q, k, v, H, D ** -0.5, w2, g, "max", emulate=False)
    assert (a - ref_a).abs().max().item() <= 2e-3 * ref_a.abs().max().item()
    assert (b - ref_b).abs().max().item() <= 2e-3 * ref_b.abs().max().item()


@pytest.mark.parametrize("B,N,H,grid,idx", [
    (2, 4096, 8, 0, [0, -1]), (2, 4096, 8, 0, [-1, 0]), (16, 4096, 8, 0, [v for i in range(8) for v in (i, -1)]),
    (16, 2048, 8, 0, list(range(8)) + [-1] * 8), (3, 1024, 5, 0, [0, 1, -1]), (4, 640, 3, 20, [-1, -1, -1, 0]),
    (5, 384, 10, 7, [0, 1, 2, 3, 4]), (4, 1024, 8, 8, [0, -1, 1, -1]), (2, 1024, 8, 3, [0, -1]), (5, 333, 3, 4, [0, -1, 1, -1, 2]),
    (1, 100, 1, 0, [0])])
def test_grouped_head_job_table_built_on_the_device_equals_the_host_replay(B, N, H, grid, idx):
    """The grouped-head kernel (head dim 40) builds every CTA's job table in shared memory with ballots and warp scans;
    the library's host replay walks the same lists sequentially (tests/test_fused2_schedule.py checks ITS invariants).
    Dump the device tables and compare them job by job."""
    import ctypes
    L = _native.lib()
    D, T, G = 40, 77, L.pww_debug_fused2_heads_per_unit()
    q, k, v, w = _inputs(B, N, H, D, T, seed=B + N + H)
    nbw = max(idx) + 1
    tiles = (N + 127) // 128
    hg = (H + G - 1) // G
    units = B * hg * tiles
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = min(units, sms if grid == 0 else min(grid, sms))
    dump = torch.zeros(g * (2 + 1024), dtype=torch.int32, device="cuda")
    L.pww_debug_set_fused_jobs_dump.argtypes = [ctypes.c_void_p]
    _set_fused_grid(grid)
    L.pww_debug_set_fused_jobs_dump(dump.data_ptr())
    try:
        _run(q, k, v, H, D ** -0.5, w[:nbw].contiguous(), 0.5, "max", torch.tensor(idx, dtype=torch.int32))
    finally:
        L.pww_debug_set_fused_jobs_dump(None)
        _set_fused_grid(0)
    d = dump.cpu().numpy().astype(np.int64).reshape(g, 2 + 1024)
    L.pww_debug_fused2_schedule.restype = ctypes.c_int
    L.pww_debug_fused2_schedule.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    widx = np.asarray(idx, dtype=np.int32)
    cap = 2 * B * H * tiles + 8
    out = np.full((cap, 14), -7, dtype=np.int32)
    n = L.pww_debug_fused2_schedule(B, H, G, tiles, g, widx.ctypes.data, out.ctypes.data, cap)
    assert n > 0
    host = out[:n]
    for cta in range(g):
        rows = host[host[:, 0] == cta]
        njobs, ns = int(d[cta, 0]), int(d[cta, 1])
        assert njobs == len(rows) and ns == int((rows[:, 2] == 0).sum())
        for r in rows:
            i = int(r[1])
            x, y = int(d[cta, 2 + 2 * i]) & 0xFFFFFFFF, int(d[cta, 3 + 2 * i]) & 0xFFFFFFFF
            assert (x & 0xFF, (x >> 8) & 0xFF, x >> 16) == (r[4], r[5], r[6]), (cta, i)
            assert (y & 1, (y >> 1) & 1, (y >> 2) & 1, (y >> 3) & 1) == (r[2], r[7], r[12], r[13]), (cta, i)
            assert ((y >> 8) & 0xFF) == r[11]
            if r[7]:
                assert ((y >> 4) & 3) == r[8]
