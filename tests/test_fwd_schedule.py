"""CPU checks of the cross-attention forward kernel's unit schedule (csrc/xattn_tc.cuh: FwdWalk, cta_range), replayed on
the host by the library itself (pww_debug_fwd_schedule runs the same code the kernel compiles).  The reference has no
counterpart: it loops heads inside one bmm (paint_with_words.py:83-118); what must hold is that every (image, head, row
tile) is computed exactly once and that every CTA gets the same mix of biased and unbiased units.  Unit record: cta,
it, b, h, tile."""
import ctypes
import itertools

import numpy as np
import pytest

from paint_with_words_sd_b200 import _native


def _schedule(B, H, tiles, grid, widx):
    L = _native.lib()
    L.pww_debug_fwd_schedule.restype = ctypes.c_int
    L.pww_debug_fwd_schedule.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_void_p]
    w = np.asarray(widx, dtype=np.int32)
    out = np.full((B * H * tiles, 5), -7, dtype=np.int32)
    n = L.pww_debug_fwd_schedule(B, H, tiles, grid, w.ctypes.data, out.ctypes.data)
    assert n == B * H * tiles
    return out


CASES = [
    (2, 8, 32, 148, [0, -1]),                      # the workload: cond + uncond, SD1.5 64x64 latents
    (2, 8, 32, 148, [-1, 0]),
    (16, 8, 32, 148, list(range(8)) + [-1] * 8),   # batched CFG, conditional half first
    (16, 8, 32, 148, [-1] * 8 + list(range(8))),
    (16, 8, 32, 148, [v for i in range(8) for v in (i, -1)]),
    (3, 5, 72, 148, [0, 1, -1]),                   # odd head count (SD2.1), one biased image without a partner
    (4, 20, 5, 148, [-1, -1, -1, 0]),
    (1, 8, 32, 148, [0]),                          # reference-style single call
    (1, 8, 1, 148, [-1]),                          # fewer units than CTAs
    (5, 10, 3, 7, [0, 1, 2, 3, 4]),                # all biased
    (33, 8, 2, 148, [(-1 if i % 3 else i // 3) for i in range(33)]),
    # the same launches on the H100's 132 SMs
    (2, 8, 32, 132, [0, -1]),
    (16, 8, 32, 132, [v for i in range(8) for v in (i, -1)]),
    (3, 5, 72, 132, [0, 1, -1]),
]


@pytest.mark.parametrize("B,H,tiles,grid,widx", CASES)
def test_every_unit_once(B, H, tiles, grid, widx):
    s = _schedule(B, H, tiles, grid, widx)
    # every (image, head, tile) exactly once
    keys = set(map(tuple, s[:, 2:5].tolist()))
    assert len(keys) == B * H * tiles
    assert keys == set(itertools.product(range(B), range(H), range(tiles)))
    for cta in np.unique(s[:, 0]):
        rows = s[s[:, 0] == cta]
        assert rows[:, 1].tolist() == list(range(len(rows)))          # contiguous iterations


@pytest.mark.parametrize("order", ["cond_first", "uncond_first", "interleaved"])
def test_cfg_units_are_balanced_whatever_the_image_order(order):
    B, H, tiles, grid = 16, 8, 32, 132
    widx = {"cond_first": list(range(8)) + [-1] * 8, "uncond_first": [-1] * 8 + list(range(8)),
            "interleaved": [v for i in range(8) for v in (i, -1)]}[order]
    s = _schedule(B, H, tiles, grid, widx)
    for cta in range(grid):
        rows = s[s[:, 0] == cta]
        nb = sum(widx[b] >= 0 for b in rows[:, 2])
        assert abs(2 * nb - len(rows)) <= 2, (cta, nb, len(rows))     # biased and unbiased units alternate
        # both operand stages (even / odd iterations) get the same mix
        for par in (0, 1):
            sub = rows[rows[:, 1] % 2 == par]
            nbp = sum(widx[b] >= 0 for b in sub[:, 2])
            assert abs(2 * nbp - len(sub)) <= 2
