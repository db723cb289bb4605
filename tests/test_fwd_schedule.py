"""CPU checks of the cross-attention forward kernel's unit schedule (csrc/xattn_tc.cuh: FwdWalk, cta_range,
mask_release_pos), replayed on the host by the library itself (pww_debug_fwd_schedule runs the same code the kernel
compiles).  The reference has no counterpart: it loops heads inside one bmm (paint_with_words.py:83-118); what must hold
is that every (image, head, row tile) is computed exactly once and that the shared mask tile protocol cannot hang or
be released early."""
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
    out = np.full((B * H * tiles, 8), -7, dtype=np.int32)
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
def test_every_unit_once_and_mask_protocol(B, H, tiles, grid, widx):
    s = _schedule(B, H, tiles, grid, widx)
    # every (image, head, tile) exactly once
    keys = set(map(tuple, s[:, 2:5].tolist()))
    assert len(keys) == B * H * tiles
    assert keys == set(itertools.product(range(B), range(H), range(tiles)))
    for cta in np.unique(s[:, 0]):
        rows = s[s[:, 0] == cta]
        assert rows[:, 1].tolist() == list(range(len(rows)))          # contiguous iterations
        for grp in np.unique(rows[:, 5]):
            g = rows[rows[:, 5] == grp]
            assert (g[:, 7] & 1).sum() == 1, "every softmax warp releases the mask tile exactly once per group"
            rel = int(np.argmax(g[:, 7] & 1))
            # phase rule of the mask barrier: every softmax warp (both groups) waits for B_MFULL exactly once per
            # group, at the group's first unit in this CTA -> each warp observes phases 0, 1, 2, ... in order and
            # arrives on B_MEMPTY only after it has observed the phase it releases
            assert ((g[:, 7] >> 1) & 1).tolist() == [1] + [0] * (len(g) - 1)
            assert int(np.argmax((g[:, 7] >> 1) & 1)) <= rel
            biased = [i for i, r in enumerate(g) if widx[r[2]] >= 0]
            for i in biased:
                assert g[i, 6] == g[i, 2], "a biased unit must find its own image's mask tile staged"
                assert i <= rel, "no mask read after the tile was released"
            assert len(set(g[:, 4].tolist())) == 1 and len(set(g[:, 6].tolist())) == 1   # one tile, one mask per group


@pytest.mark.parametrize("order", ["cond_first", "uncond_first", "interleaved"])
def test_cfg_batches_are_balanced_whatever_the_image_order(order):
    B, H, tiles, grid = 16, 8, 32, 132
    widx = {"cond_first": list(range(8)) + [-1] * 8, "uncond_first": [-1] * 8 + list(range(8)),
            "interleaved": [v for i in range(8) for v in (i, -1)]}[order]
    s = _schedule(B, H, tiles, grid, widx)
    for cta in range(grid):
        rows = s[s[:, 0] == cta]
        nb = sum(widx[b] >= 0 for b in rows[:, 2])
        assert abs(2 * nb - len(rows)) <= 2, (cta, nb, len(rows))     # biased and unbiased units alternate
        # both softmax groups (even / odd iterations) get the same mix
        for par in (0, 1):
            sub = rows[rows[:, 1] % 2 == par]
            nbp = sum(widx[b] >= 0 for b in sub[:, 2])
            assert abs(2 * nbp - len(sub)) <= 2


def _waited_phases_old_rule(rows, widx, group):
    """Round-1 rule (the bug): a softmax group waited for B_MFULL only at ITS OWN units that read the mask."""
    return [int(r[5]) for r in rows if r[1] % 2 == group and widx[r[2]] >= 0 and r[6] >= 0]


def test_old_wait_rule_skipped_phases_and_new_rule_does_not():
    """Round 1 failed test_bias_path_matches_oracle[max-4096-8-40] intermittently: a softmax group whose first
    mask-reading unit lay in the CTA's SECOND mask group waited for parity 1 of B_MFULL without having observed
    phase 0, so the parity test could pass before the first tile had landed.  The replay shows the old rule skipped
    phases on some CTAs of exactly that launch, and that under the new rule every warp waits on every phase."""
    B, H, tiles, grid, widx = 1, 8, 32, 132, [0]
    s = _schedule(B, H, tiles, grid, widx)
    exposed = []
    for cta in range(grid):
        rows = s[s[:, 0] == cta]
        ngroups = len(np.unique(rows[:, 5]))
        for group in (0, 1):
            old = sorted(set(_waited_phases_old_rule(rows, widx, group)))
            if old and old != list(range(old[-1] + 1)):
                exposed.append(cta)
        new = [int(r[5]) for r in rows if (r[7] >> 1) & 1]
        assert new == list(range(ngroups)), (cta, new)
    assert exposed, "the replay must reproduce the round-1 hazard under the old rule"
