"""CPU checks of the one-launch kernel's job lists (csrc/xattn_fused2.cuh: Fx2Jobs over FxWalk with head groups), replayed
on the host by the library itself (the same code the kernel's host-replay test compares the device-built tables with).
What must hold: every (image, head, row tile) is a softmax job exactly once; every unit of an image with a weight map is
a statistic job exactly once, before any softmax job of its CTA; the unbiased softmax jobs of a CTA precede its biased
ones (they overlap the grid barrier); the jobs of a unit are consecutive heads of one head group; a CTA's jobs cover
exactly the units of its range; the set of CTAs the barrier of image b waits for is exactly the set that publishes a
partial for b.  Job record: cta, i, kind (0 = stat, 1 = softmax), b, h, tile, biased, li."""
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
    out = np.full((cap, 8), -7, dtype=np.int32)
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


def _unit_passes(rows):
    """Split a CTA's jobs into unit passes: maximal runs of consecutive jobs of one (kind, image, tile, head group)."""
    runs = []
    for r in rows:
        key = (r[2], r[3], r[5], r[4] // G)
        if runs and runs[-1][0] == key:
            runs[-1][1].append(r)
        else:
            runs.append((key, [r]))
    return [np.array(r) for _, r in runs]


@pytest.mark.parametrize("B,H,tiles,grid,widx", CASES)
def test_job_lists_cover_every_unit_once(B, H, tiles, grid, widx):
    j = _jobs(B, H, tiles, grid, widx)
    main, stat = j[j[:, 2] == 1], j[j[:, 2] == 0]
    units = set(itertools.product(range(B), range(H), range(tiles)))
    assert len(main) == len(units) and set(map(tuple, main[:, 3:6].tolist())) == units
    biased = {u for u in units if widx[u[0]] >= 0}
    assert len(stat) == len(biased) and set(map(tuple, stat[:, 3:6].tolist())) == biased
    assert (j[:, 6] == np.array([widx[b] >= 0 for b in j[:, 3]])).all()
    hg = (H + G - 1) // G
    total_units = B * hg * tiles
    for cta in np.unique(j[:, 0]):
        rows = j[j[:, 0] == cta]
        u0, u1 = cta * total_units // grid, (cta + 1) * total_units // grid
        assert rows[:, 1].tolist() == list(range(len(rows)))
        kinds = rows[:, 2].tolist()
        assert kinds == sorted(kinds)
        m = rows[rows[:, 2] == 1]
        flags = m[:, 6].tolist()
        assert flags == sorted(flags)
        sb = rows[rows[:, 2] == 0][:, [3, 4, 5, 7]].tolist()
        mb = m[m[:, 6] == 1][:, [3, 4, 5, 7]].tolist()
        assert sb == mb                                                    # same units and local image in both passes
        if sb:
            li = [r[3] for r in sb]
            assert li[0] == 0 and all(b - a in (0, 1) for a, b in zip(li, li[1:])) and max(li) < K_MAX_LOCAL
        # the heads of a unit are consecutive jobs, grouped by G
        passes = _unit_passes(rows)
        assert len(passes) == len({(k, b, h // G, t) for k, b, h, t in rows[:, 2:6].tolist()})
        for r in passes:
            heads = r[:, 4].tolist()
            assert heads == list(range(heads[0], heads[0] + len(heads))) and heads[0] % G == 0
            assert len(heads) == min(G, H - heads[0])
        # every unit of the range is visited: distinct (image, head group, tile) == number of units
        assert len({(b, h // G, t) for b, h, t in m[:, 3:6].tolist()}) == u1 - u0
    # grid barrier membership: the CTAs image b's waiters expect == the CTAs that run a statistic job of image b
    for b in range(B):
        if widx[b] < 0:
            continue
        publishers = set(stat[stat[:, 3] == b][:, 0].tolist())
        expected = {c for c in range(grid) if _has_image(c, grid, B, H, tiles, widx, b)}
        assert publishers == expected, (b, sorted(publishers ^ expected))


def test_the_workload_launch_holds_two_units_per_cta():
    """cond + uncond at N = 4096, 8 heads on 132 CTAs (one per H100 SM): at most two units per CTA; with 2 heads per unit
    most CTAs hold one biased and one unbiased unit, whose softmax jobs overlap the grid barrier."""
    hg = (8 + G - 1) // G
    grid = min(132, 2 * 32 * hg)
    j = _jobs(2, 8, 32, grid, [0, -1])
    both = 0
    for cta in range(grid):
        rows = j[j[:, 0] == cta]
        assert len({(b, h // G, t) for b, h, t in rows[:, 3:6].tolist()}) <= 2
        kinds = set(map(tuple, rows[rows[:, 2] == 1][:, [6]].tolist()))
        both += len(kinds) == 2
    if G == 2:
        assert both >= 100
