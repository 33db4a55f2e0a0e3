"""CPU tests of the chain's TRAA frame tail (rfx_ssgi_chain_enable_traa): the ctypes mirror of rfx_traa_tail_options has the C layout,
and the row ranges of a row-sharded frame with the tail (rfx_shard_ranges with n_launches = 4 + n_poisson) equal the Python mirror
(ShardPlan(traa=True)) while the ranges without the tail stay what they were."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

from realism_effects_b200 import abi
from realism_effects_b200.parallel import ShardPlan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_traa_tail_options_layout_matches_c(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rfx.h"\nint main(void){printf("%zu %zu %zu\\n", sizeof(rfx_traa_tail_options), '
                   'offsetof(rfx_traa_tail_options, max_blend), offsetof(rfx_traa_tail_options, full_accumulate)); return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, off_blend, off_full = (int(x) for x in subprocess.check_output([str(exe)], text=True).split())
    assert size == C.sizeof(abi.TraaTailOptions)
    assert off_blend == abi.TraaTailOptions.max_blend.offset and off_full == abi.TraaTailOptions.full_accumulate.offset


def test_traa_defaults_are_what_traa_effect_forces():
    o = abi.make_traa_tail_options()
    assert (o.max_blend, o.neighborhood_clamp_intensity, o.confidence_power, o.log_transform, o.full_accumulate) == (np.float32(0.9), 1.0, 4.0, 1, 0)
    assert o.compose.use_fog == 0 and o.compose.is_debug == 0


def test_tail_rows_constant_matches_the_header():
    hdr = open(os.path.join(ROOT, "include", "rfx.h")).read()
    assert int(re.search(r"#define RFX_TRAA_TAIL_ROWS (\d+)", hdr).group(1)) == ShardPlan.TRAA_TAIL_ROWS == 4


def _native(lib, W, H, r0, r1, passes, radius, n):
    out = (C.c_uint32 * (2 * n))()
    st = lib.rfx_shard_ranges(W, H, r0, r1, passes, radius, 1, out, n)
    return st, [(out[2 * k], out[2 * k + 1]) for k in range(n)]


def test_native_ranges_with_the_tail_match_the_mirror(built):
    """2..8 bands, landscape and portrait, borders moved off the equal split: rfx_shard_ranges(n = 4 + passes) == ShardPlan(traa=True)"""
    lib = abi.lib()
    for W, H, passes, radius in ((3840, 2160, 4, 3.0), (540, 960, 2, 3.0), (7680, 4320, 4, 11.0), (320, 592, 4, 3.0), (256, 512, 0, 3.0)):
        for world in range(2, 9):
            base = [int(round(H * i / world / 16.0)) * 16 for i in range(world)] + [H]
            for shift in (0, 16, -16):
                bounds = tuple([0] + [b + shift for b in base[1:-1]] + [H])
                for rank in range(world):
                    p = ShardPlan(H, world, rank, passes, radius, True, bounds=bounds, width=W, traa=True)
                    assert p.n_launches == 4 + passes
                    st, got = _native(lib, W, H, p.r0, p.r1, passes, radius, p.n_launches)
                    assert st == 0 and got == p.ranges, (W, H, world, shift, rank)
                    plain = ShardPlan(H, world, rank, passes, radius, True, bounds=bounds, width=W)
                    st, got0 = _native(lib, W, H, p.r0, p.r1, passes, radius, plain.n_launches)
                    assert st == 0 and got0 == plain.ranges
                    # the tail runs on the band; K4 widens by the tail's rows; every earlier launch contains the one after it
                    assert p.ranges[-1] == (p.r0, p.r1)
                    assert p.ranges[-2] == (max(0, p.r0 - 4), min(H, p.r1 + 4))
                    for k in range(len(p.ranges) - 1):
                        assert p.ranges[k][0] <= p.ranges[k + 1][0] and p.ranges[k][1] >= p.ranges[k + 1][1]


def test_native_ranges_without_the_tail_are_unchanged(built):
    """n_launches = 3 + passes keeps today's arithmetic (K4 on the band, K3's last pass one row wider, ...)"""
    lib = abi.lib()
    st, got = _native(lib, 3840, 2160, 810, 1080, 4, 3.0, 7)
    assert st == 0
    assert got == [(791, 1099), (793, 1097), (797, 1093), (801, 1089), (805, 1085), (809, 1081), (810, 1080)]
    assert _native(lib, 3840, 2160, 810, 1080, 4, 3.0, 6)[0] != 0  # neither 3 + passes nor 4 + passes
    assert _native(lib, 3840, 2160, 810, 1080, 4, 3.0, 9)[0] != 0
