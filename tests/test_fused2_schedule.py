"""CPU checks of the one-launch kernel's job lists (csrc/xattn_fused2.cuh: Fx2Jobs over FxWalk with head groups), replayed
on the host by the library itself (the same code the kernel's host-replay test compares the device-built tables with).
What must hold: every (image, head, row tile) is a softmax job exactly once; every unit of an image with a weight map is
a statistic job exactly once, before any softmax job of its CTA; the unbiased softmax jobs of a CTA precede its biased
ones (they overlap the grid barrier); the jobs of a unit pass are consecutive, flagged first ... last, share one `up`;
`up` counts the unit passes of a CTA in order; `ul` is the unit's position in the CTA's range (the
resident stage); the set of CTAs the barrier of image b waits for is exactly the set that publishes a partial for b."""
import ctypes
import itertools

import numpy as np
import pytest

from paint_with_words_sd_b200 import _native

K_MAX_LOCAL = 4
G = _native.lib().pww_debug_fused2_heads_per_unit()      # heads per unit: a build-time constant of the library


def _jobs(B, H, tiles, grid, widx, g=G):
    L = _native.lib()
    L.pww_debug_fused2_schedule.restype = ctypes.c_int
    L.pww_debug_fused2_schedule.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    w = np.asarray(widx, dtype=np.int32)
    cap = 2 * B * H * tiles + 8
    out = np.full((cap, 14), -7, dtype=np.int32)
    n = L.pww_debug_fused2_schedule(B, H, g, tiles, grid, w.ctypes.data, out.ctypes.data, cap)
    assert n >= 0
    return out[:n]


def _has_image(cta, grid, B, H, tiles, widx, b):
    """Does CTA `cta` publish a statistic partial for image b?  (the library's membership test, head GROUPS as heads)"""
    L = _native.lib()
    L.pww_debug_fused_cta_has_image.restype = ctypes.c_int
    L.pww_debug_fused_cta_has_image.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p, ctypes.c_int]
    w = np.asarray(widx, dtype=np.int32)
    return L.pww_debug_fused_cta_has_image(cta, grid, B, (H + G - 1) // G, tiles, w.ctypes.data, b)


CASES = [
    (2, 8, 32, 128, [0, -1]),                      # the workload: 2 images x 32 tiles x 2 head groups = 128 units
    (2, 8, 32, 128, [-1, 0]),
    (16, 8, 32, 148, list(range(8)) + [-1] * 8),
    (16, 8, 32, 148, [v for i in range(8) for v in (i, -1)]),
    (3, 5, 72, 148, [0, 1, -1]),                   # 5 heads: groups of 4 + 1
    (4, 3, 5, 20, [-1, -1, -1, 0]),                # fewer heads than a group
    (1, 8, 32, 64, [0]),
    (1, 1, 1, 1, [-1]),
    (5, 10, 3, 7, [0, 1, 2, 3, 4]),
    (4, 8, 8, 8, [0, -1, 1, -1]),
    (2, 8, 8, 3, [0, -1]),
    (5, 3, 3, 4, [0, -1, 1, -1, 2]),
    # the same launches on the H100's 132 SMs
    (16, 8, 32, 132, list(range(8)) + [-1] * 8),
    (16, 8, 32, 132, [v for i in range(8) for v in (i, -1)]),
    (3, 5, 72, 132, [0, 1, -1]),
]


@pytest.mark.parametrize("B,H,tiles,grid,widx", CASES)
def test_job_lists(B, H, tiles, grid, widx):
    j = _jobs(B, H, tiles, grid, widx)
    main, stat = j[j[:, 2] == 1], j[j[:, 2] == 0]
    units = set(itertools.product(range(B), range(H), range(tiles)))
    assert len(main) == len(units) and set(map(tuple, main[:, 4:7].tolist())) == units
    biased = {u for u in units if widx[u[0]] >= 0}
    assert len(stat) == len(biased) and set(map(tuple, stat[:, 4:7].tolist())) == biased
    hg = (H + G - 1) // G
    total_units = B * hg * tiles
    for cta in np.unique(j[:, 0]):
        rows = j[j[:, 0] == cta]
        u0, u1 = cta * total_units // grid, (cta + 1) * total_units // grid
        assert rows[:, 1].tolist() == list(range(len(rows)))
        kinds = rows[:, 2].tolist()
        assert kinds == sorted(kinds)
        m = rows[rows[:, 2] == 1]
        assert m[:, 3].tolist() == list(range(len(m)))
        flags = m[:, 7].tolist()
        assert flags == sorted(flags)
        sb = rows[rows[:, 2] == 0][:, [4, 5, 6, 8, 11]].tolist()
        mb = m[m[:, 7] == 1][:, [4, 5, 6, 8, 11]].tolist()
        assert sb == mb                                                    # same units, local image and stage in both passes
        if sb:
            li = [r[3] for r in sb]
            assert li[0] == 0 and all(b - a in (0, 1) for a, b in zip(li, li[1:])) and max(li) < K_MAX_LOCAL
        # unit passes: consecutive jobs, first/last flags, one `up` each, counting up; `ul` inside the CTA's range
        ups = rows[:, 10].tolist()
        assert ups == sorted(ups) and ups[0] == 0 and set(ups) == set(range(max(ups) + 1))
        for up in set(ups):
            r = rows[rows[:, 10] == up]
            assert r[0, 12] == 1 and r[-1, 13] == 1 and r[1:, 12].sum() == 0 and r[:-1, 13].sum() == 0
            assert len(set(map(tuple, r[:, [2, 4, 6, 7, 11]].tolist()))) == 1          # one pass of one unit
            heads = r[:, 5].tolist()
            assert heads == list(range(heads[0], heads[0] + len(heads))) and heads[0] % G == 0
            assert len(heads) == min(G, H - heads[0])
            assert 0 <= r[0, 11] < u1 - u0
        # every unit of the range is visited: distinct (ul) values == number of units
        assert set(rows[:, 11].tolist()) == set(range(u1 - u0))
    # grid barrier membership: the CTAs image b's waiters expect == the CTAs that run a statistic job of image b
    for b in range(B):
        if widx[b] < 0:
            continue
        publishers = set(stat[stat[:, 4] == b][:, 0].tolist())
        expected = {c for c in range(grid) if _has_image(c, grid, B, H, tiles, widx, b)}
        assert publishers == expected, (b, sorted(publishers ^ expected))


def test_the_workload_launch_is_resident():
    """cond + uncond at N = 4096, 8 heads on 132 CTAs (one per H100 SM): at most two units per CTA; with 2 heads per unit
    most CTAs hold one biased and one unbiased unit, whose softmax jobs overlap the grid barrier."""
    hg = (8 + G - 1) // G
    grid = min(132, 2 * 32 * hg)
    j = _jobs(2, 8, 32, grid, [0, -1])
    both = 0
    for cta in range(grid):
        rows = j[j[:, 0] == cta]
        assert set(rows[:, 11].tolist()) <= {0, 1}
        kinds = set(map(tuple, rows[rows[:, 2] == 1][:, [7]].tolist()))
        both += len(kinds) == 2
    if G == 2:
        assert both >= 100
