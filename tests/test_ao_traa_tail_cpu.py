"""The AO chain's TRAA frame tail, host side: rfx_ao_shard_ranges with the tail (n_launches = 3 + 2 * iterations) against its Python
mirror parallel.AoShardPlan(traa=True), the containment of every row the tail reads of the K7 plane (K2's 5x5 LINEAR clamp window on the
band +- 1, K9's LINEAR fetch of the accumulated plane) in K7's range, today's ranges without the tail, and the ctypes mirror of
rfx_ao_traa_frame.  No GPU needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from realism_effects_b200 import abi, parallel
from test_ao_group_cpu import _rows_read, bands

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(640, 360), (300, 520), (333, 257)]
SIZE_IDS = ["landscape", "portrait", "odd"]


def c_ranges(W, H, own, iterations, radius, n):
    out = (C.c_uint32 * (2 * n))()
    st = abi.lib().rfx_ao_shard_ranges(W, H, own[0], own[1], iterations, radius, out, n)
    return st, [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


@pytest.mark.parametrize("iterations", [0, 1, 2, 3])
@pytest.mark.parametrize("radius", [3.0, 11.0, 32.0])
@pytest.mark.parametrize("size", SIZES, ids=SIZE_IDS)
def test_c_ranges_with_the_tail_equal_the_python_plan(built, iterations, radius, size):
    W, H = size
    for n in range(2, 9):
        for shift in (0, 16, -16, 5):
            b = bands(H, n, shift)
            for r in range(n):
                own = (b[r], b[r + 1])
                plan = parallel.AoShardPlan(W, H, own, iterations, radius, traa=True)
                assert plan.n_launches == 3 + 2 * iterations
                st, got = c_ranges(W, H, own, iterations, radius, plan.n_launches)
                assert st == abi.RFX_OK and got == plan.ranges, (size, n, shift, r)
                assert got[-1] == own  # the tail runs on the band
                assert got[-2] == (max(0, own[0] - 4), min(H, own[1] + 4))  # K7 on the band +- RFX_TRAA_TAIL_ROWS
                # every earlier launch widens from K7's range exactly as the chain without the tail widens from the band
                st, plain = c_ranges(W, H, got[-2], iterations, radius, 2 + 2 * iterations)
                assert st == abi.RFX_OK and plain == got[:-1]


def _tail_rows_read(H, band):
    """rows of the K7 plane the tail reads for the output rows `band`: K9 fetches the accumulated plane LINEAR at the pixel centre, so K2
    runs on the band +- 1; K2 fetches K7 LINEAR at vUv + (0, dy) / H for |dy| <= 2 (the clamp window); clamp-to-edge keeps rows in the frame"""
    y = np.arange(max(0, band[0] - 1), min(H, band[1] + 1), dtype=np.float64)
    k2_rows = (int(y.min()), int(y.max()) + 1)
    acc = _rows_read(0, H, band, 0.0, k7=True)  # K9's LINEAR fetch of the accumulated plane at the pixel centre
    assert k2_rows[0] <= acc[0] and acc[1] < k2_rows[1]
    lo, hi = H, -1
    for dy in range(-2, 3):
        t = ((y + 0.5) / H + dy / H) * H - 0.5
        lo, hi = min(lo, int(np.floor(t.min()))), max(hi, int(np.floor(t.max())) + 1)
    return max(0, lo), min(H - 1, hi)


@pytest.mark.parametrize("iterations", [0, 1, 2])
@pytest.mark.parametrize("size,radius", [((640, 360), 3.0), ((300, 520), 11.0), ((333, 257), 32.0)])
def test_every_row_a_launch_reads_lies_in_the_earlier_launch_range(built, iterations, size, radius):
    W, H = size
    for n in (2, 4, 5):
        b = bands(H, n, 16 if n < 5 else 5)
        for r in range(n):
            own = (b[r], b[r + 1])
            st, rng = c_ranges(W, H, own, iterations, radius, 3 + 2 * iterations)
            assert st == abi.RFX_OK
            lo, hi = _tail_rows_read(H, rng[-1])
            assert rng[-2][0] <= lo and hi < rng[-2][1], (size, n, r, (lo, hi), rng[-2])
            for k in range(1, len(rng) - 1):  # K3 passes and K7 read their inputs as without the tail
                lo, hi = _rows_read(W, H, rng[k], radius, k7=(k == len(rng) - 2))
                assert rng[k - 1][0] <= lo and hi < rng[k - 1][1], (size, n, r, k, (lo, hi), rng[k - 1])


def test_ranges_without_the_tail_are_unchanged(built):
    """n_launches = 2 + 2 * iterations keeps today's arithmetic; every other count is refused"""
    st, got = c_ranges(640, 360, (96, 192), 1, 3.0, 4)
    assert st == abi.RFX_OK and got == [(87, 201), (91, 197), (95, 193), (96, 192)]
    for W, H in SIZES:
        for it in range(4):
            own = (H // 3, 2 * H // 3)
            assert c_ranges(W, H, own, it, 11.0, 2 + 2 * it) == (abi.RFX_OK, parallel.AoShardPlan(W, H, own, it, 11.0).ranges)
            for n in (1 + 2 * it, 4 + 2 * it):
                assert c_ranges(W, H, own, it, 11.0, n)[0] == 1, (it, n)


def test_ctypes_mirror_of_the_ao_traa_frame_matches_c(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rfx.h"\nint main(void){printf("%zu %zu %zu\\n", sizeof(rfx_ao_traa_frame), '
                   'offsetof(rfx_ao_traa_frame, camera_pos), offsetof(rfx_ao_traa_frame, camera_moved)); return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, off_pos, off_moved = (int(x) for x in subprocess.check_output([str(exe)], text=True).split())
    assert size == C.sizeof(abi.AoTraaFrame)
    assert off_pos == abi.AoTraaFrame.camera_pos.offset and off_moved == abi.AoTraaFrame.camera_moved.offset


def test_the_new_entry_points_are_exported(built):
    lib = abi.lib()
    for name in ("rfx_ao_chain_enable_traa", "rfx_ao_chain_render_traa", "rfx_ao_chain_render_sharded_traa"):
        assert name in abi.EXPORTS and hasattr(lib, name)
