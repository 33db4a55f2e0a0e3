"""CPU tests of the row ranges a group plans for every denoise mode: denoiseMode "full_temporal" / "temporal" run no Poisson pass, so their
frame uses the ranges of rfx_shard_ranges with n_poisson_passes = 0 (K1, K2, K4, and the TRAA tail when it is on), mirrored by
ShardPlan(denoise_mode=...), and K1 / K2 are widened only by the launches that run.  The ranges of denoiseMode "full" are unchanged."""
import ctypes as C

from realism_effects_b200 import abi
from realism_effects_b200.parallel import ShardPlan

FULL, FULL_TEMPORAL, TEMPORAL = 0, 1, 2
SIZES = ((3840, 2160, 4, 3.0), (540, 960, 2, 3.0), (7680, 4320, 4, 11.0), (320, 592, 4, 3.0), (256, 512, 0, 3.0))


def _native(lib, W, H, r0, r1, passes, radius, n):
    out = (C.c_uint32 * (2 * n))()
    st = lib.rfx_shard_ranges(W, H, r0, r1, passes, radius, 1, out, n)
    return st, [(out[2 * k], out[2 * k + 1]) for k in range(n)]


def _plans():
    """every band of 2..8 ranks, landscape and portrait, with the borders on the equal split and moved by +-16 rows"""
    for W, H, passes, radius in SIZES:
        for world in range(2, 9):
            base = [int(round(H * i / world / 16.0)) * 16 for i in range(world)] + [H]
            for shift in (0, 16, -16):
                bounds = tuple([0] + [b + shift for b in base[1:-1]] + [H])
                for rank in range(world):
                    yield W, H, passes, radius, world, bounds, rank


def test_native_ranges_match_the_mirror_in_every_denoise_mode(built):
    lib = abi.lib()
    for W, H, passes, radius, world, bounds, rank in _plans():
        for dm in (FULL, FULL_TEMPORAL, TEMPORAL):
            for traa in (False, True):
                p = ShardPlan(H, world, rank, passes, radius, True, bounds=bounds, width=W, traa=traa, denoise_mode=dm)
                native_passes = passes if dm == FULL else 0
                assert p.passes == native_passes
                assert p.n_launches == 3 + native_passes + (1 if traa else 0)
                st, got = _native(lib, W, H, p.r0, p.r1, native_passes, radius, p.n_launches)
                assert st == 0 and got == p.ranges, (W, H, world, rank, dm, traa)


def test_temporal_modes_widen_k1_and_k2_only_by_the_launches_that_run(built):
    """full_temporal / temporal: K2 covers K4's range (or, with the tail, the tail's band + RFX_TRAA_TAIL_ROWS) and K1 adds the 5x5 window
    of K2 - no Poisson halo - and K4 itself is the band (no Poisson pass feeds it)."""
    for W, H, passes, radius, world, bounds, rank in _plans():
        for dm in (FULL_TEMPORAL, TEMPORAL):
            for traa in (False, True):
                p = ShardPlan(H, world, rank, passes, radius, True, bounds=bounds, width=W, traa=traa, denoise_mode=dm)
                k1, k2, k4 = p.ranges[:3]
                own = (p.r0, p.r1)
                widen = lambda r, n: (max(0, r[0] - n), min(H, r[1] + n))  # noqa: E731
                assert k4 == (widen(own, ShardPlan.TRAA_TAIL_ROWS) if traa else own)
                assert k2 == k4
                assert k1 == widen(k4, ShardPlan.K2_NEIGHBOURHOOD_ROWS)
                assert k1[0] >= widen(k4, ShardPlan.K2_NEIGHBOURHOOD_ROWS + ShardPlan.K4_INPUT_ROWS)[0]
                assert k1[1] <= widen(k4, ShardPlan.K2_NEIGHBOURHOOD_ROWS + ShardPlan.K4_INPUT_ROWS)[1]
                if traa:
                    assert p.ranges[3] == own


def test_full_mode_ranges_are_unchanged(built):
    """denoise_mode defaults to "full": the existing arguments give the existing ranges"""
    lib = abi.lib()
    p = ShardPlan(2160, 8, 3, 4, 3.0, True, bounds=(0, 270, 540, 810, 1080, 1350, 1620, 1890, 2160), width=3840)
    assert p.ranges == [(791, 1099), (793, 1097), (797, 1093), (801, 1089), (805, 1085), (809, 1081), (810, 1080)]
    assert _native(lib, 3840, 2160, 810, 1080, 4, 3.0, 7) == (0, p.ranges)
    assert ShardPlan(2160, 8, 3, 4, 3.0, True, bounds=p.bounds, width=3840, denoise_mode=FULL).ranges == p.ranges
