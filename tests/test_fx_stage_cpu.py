"""The cosmetic stage of the TRAA tail (rfx_*_chain_set_effects), host side: the rows of the tail's image the stage reads around a band
(rfx_fx_stage_rows) equal the Python mirror (parallel.fx_stage_rows / lens_rows) and contain every tap footprint of a brute-force float32
evaluation of the effects' fetches, and the launch ranges of a row-sharded frame with the stage (ShardPlan / AoShardPlan with stage_rows)
are those the chains plan: rfx_shard_ranges / rfx_ao_shard_ranges over the stage's rows, then the band for the stage."""
import ctypes as C

import numpy as np
import pytest

from realism_effects_b200 import abi, parallel
from realism_effects_b200.parallel import AoShardPlan, ShardPlan

ERR_INVALID_ARG = 1  # include/rfx.h RFX_ERR_INVALID_ARG
S, L, G, SP = abi.FX_SHARPNESS, abi.FX_LENS_DISTORTION, abi.FX_GRADUAL_BACKGROUND, abi.FX_SPARKLE
SIZES = [(640, 360), (360, 640), (333, 197), (333, 198)]
EFFECT_LISTS = [[S], [L], [G], [SP], [S, G], [L, S, G, SP], [G, SP, S, L]]
# the defaults, strong barrel, strong pincushion (1 - alpha * q crosses 0 inside the frame), and alpha 4, which puts 1 - alpha * r at
# exactly 0 on the centre column of odd widths (333 x 198: X = 0, Y = -0.5 on row 49): 0 / 0 there, a non-finite uv
LENS = [(-0.05, -0.05, 1.0), (-0.3, -0.3, 1.0), (0.3, 0.3, 1.0), (0.3, -0.3, 2.5), (4.0, 4.0, 1.0)]


def bands(H):
    return [(0, H // 4), (H // 3, 2 * H // 3), (3 * H // 4, H), (H // 2, H // 2 + 16)]


def params(effects, lens=(-0.05, -0.05, 1.0)):
    p = abi.EffectsParams()
    p.n_effects = len(effects)
    for i, e in enumerate(effects):
        p.effects[i] = e
    p.sharpness = 0.75
    p.alphax, p.alphay, p.aberration = lens
    return p


def native_rows(W, H, p, own):
    rows = (C.c_uint32 * 2)()
    st = abi.lib().rfx_fx_stage_rows(W, H, C.byref(p), own[0], own[1], rows)
    return st, (int(rows[0]), int(rows[1]))


def test_native_stage_rows_equal_the_mirror(built):
    for W, H in SIZES:
        for lens in LENS:
            for effects in EFFECT_LISTS:
                for own in bands(H):
                    st, got = native_rows(W, H, params(effects, lens), own)
                    assert st == abi.RFX_OK
                    assert got == parallel.fx_stage_rows(W, H, own, effects, *lens), (W, H, lens, effects, own)


def test_stage_rows_without_lens_distortion_are_the_fixed_reach(built):
    W, H = 640, 360
    for own in bands(H):
        assert native_rows(W, H, params([G, SP]), own)[1] == (max(0, own[0] - 1), min(H, own[1] + 1))
        assert native_rows(W, H, params([SP, S]), own)[1] == (max(0, own[0] - 2), min(H, own[1] + 2))


def test_bad_arguments_are_refused(built):
    lib = abi.lib()
    rows = (C.c_uint32 * 2)()
    assert native_rows(640, 360, params([]), (0, 90))[0] == ERR_INVALID_ARG
    p = params([S])
    p.effects[0] = 9
    assert native_rows(640, 360, p, (0, 90))[0] == ERR_INVALID_ARG
    assert native_rows(640, 360, params([S]), (90, 90))[0] == ERR_INVALID_ARG
    assert native_rows(640, 360, params([S]), (0, 361))[0] == ERR_INVALID_ARG
    assert lib.rfx_fx_stage_rows(640, 360, None, 0, 90, rows) == ERR_INVALID_ARG
    p = params([S])
    p.n_effects = 5
    assert native_rows(640, 360, p, (0, 90))[0] == ERR_INVALID_ARG


def _footprint(v, H):
    """rows a LINEAR fetch at v touches (bilin_setup: floor(v * H - 0.5) and the next row, clamped); None where the kernel's integer
    conversion is not exact (a non-finite or out-of-range coordinate)"""
    f = np.float32
    fy = v * f(H) - f(0.5)
    bad = ~(np.abs(fy) < f(1.0e9))
    iy = np.floor(np.where(bad, f(0.0), fy)).astype(np.int64)
    return np.clip(iy, 0, H - 1), np.clip(iy + 1, 0, H - 1), bad


def brute_force_rows(W, H, own, effects, lens):
    """every tap of every output pixel of the band, evaluated in float32 as csrc/k_fx.cu evaluates it: (lowest, highest + 1) row, or
    None when some tap coordinate is not usable (then every row is needed)"""
    f = np.float32
    one, two, half = f(1.0), f(2.0), f(0.5)
    ys = np.arange(own[0], own[1], dtype=f)
    v = ((ys + half) / f(H))[:, None] * np.ones((1, W), f)           # pixel_uv
    u = ((np.arange(W, dtype=f) + half) / f(W))[None, :] * np.ones((len(ys), 1), f)
    taps = [v]                                                       # the pass's own fetch at the pixel centre
    if S in effects:
        ts = f(1.0 / H)                                              # texelSize = 1 / size, a double rounded to fp32
        taps += [v - one * ts, v + f(-1.0) * ts, v + f(0.0) * ts, v + one * ts]
    if L in effects:
        ax, ay, ab = (f(x) for x in lens)
        with np.errstate(all="ignore"):
            x, y = (two * u - one) / one, (two * v - one) / one
            r = x * x + y * y
            x3, y3 = x / (one - ax * r), y / (one - ay * r)
            q = x3 * x3 + y3 * y3
            y2 = y / (one - ay * q)
            dv = (y2 + one) * one / two
            oy = one / f(H)
            taps += [dv - ab * f(0.0), dv - ab * oy, dv - ab * oy]
    lo, hi = H, -1
    for t in taps:
        with np.errstate(all="ignore"):
            a, b, bad = _footprint(t, H)
        if bad.any():
            return None
        lo, hi = min(lo, int(a.min())), max(hi, int(b.max()))
    return lo, hi + 1


def test_every_tap_lies_inside_the_stage_rows(built):
    for W, H in SIZES:
        for lens in LENS:
            for effects in ([S], [L], [S, L], [L, G, SP, S]):
                for own in bands(H):
                    st, (a, b) = native_rows(W, H, params(effects, lens), own)
                    assert st == abi.RFX_OK
                    need = brute_force_rows(W, H, own, effects, lens)
                    if need is None:
                        assert (a, b) == (0, H), (W, H, lens, effects, own)
                    else:
                        assert a <= need[0] and need[1] <= b, (W, H, lens, effects, own, need, (a, b))


def test_a_non_finite_uv_needs_every_row(built):
    """alpha 4 on 333 x 198: 0 / 0 on the centre column of row 49 (and its mirror row 148), so the bands holding them need the whole image"""
    W, H = 333, 198
    assert native_rows(W, H, params([L], (4.0, 4.0, 1.0)), (40, 60))[1] == (0, H)
    lo, hi = parallel.lens_rows(W, H, 4.0, 4.0, 1.0)
    assert lo[49] == 0 and hi[49] == H - 1


def test_default_lens_distortion_reaches_inward_at_the_frame_edges(built):
    """barrel distortion (the defaults) samples towards the centre: a band at the top edge reads rows below it, one in the middle no more
    than the centre fetch needs"""
    W, H = 3840, 2160
    top = native_rows(W, H, params([L]), (0, 270))[1]
    assert top[0] == 0 and top[1] > 271
    assert native_rows(W, H, params([L]), (1080 - 8, 1080 + 8))[1] == (1080 - 9, 1080 + 9)


def _shard(W, H, own, passes, radius, n):
    out = (C.c_uint32 * (2 * n))()
    st = abi.lib().rfx_shard_ranges(W, H, own[0], own[1], passes, radius, 1, out, n)
    return st, [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


def _ao_shard(W, H, own, iterations, radius, n):
    out = (C.c_uint32 * (2 * n))()
    st = abi.lib().rfx_ao_shard_ranges(W, H, own[0], own[1], iterations, radius, out, n)
    return st, [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


@pytest.mark.parametrize("effects,lens", [([S], LENS[0]), ([L], LENS[0]), ([L], LENS[2]), ([S, L, G, SP], LENS[1])])
def test_shard_plans_with_the_stage_equal_the_chains_ranges(built, effects, lens):
    """the chains plan a frame with the stage as rfx_shard_ranges / rfx_ao_shard_ranges over rfx_fx_stage_rows, then the band (the stage)"""
    for W, H in [(640, 360), (360, 640)]:
        world = 4
        b = tuple(H * i // world for i in range(world + 1))
        for rank in range(world):
            own = (b[rank], b[rank + 1])
            st, rows = native_rows(W, H, params(effects, lens), own)
            assert st == abi.RFX_OK and rows == parallel.fx_stage_rows(W, H, own, effects, *lens)
            for passes in (0, 2, 4):
                plan = ShardPlan(H, world, rank, passes, 5.0, bounds=b, width=W, traa=True, stage_rows=rows)
                st, got = _shard(W, H, rows, passes, 5.0, 4 + passes)
                assert st == abi.RFX_OK and plan.ranges == got + [own] and plan.n_launches == 5 + passes
                assert plan.ranges[-2] == rows
            for it in (0, 1, 2):
                plan = AoShardPlan(W, H, own, it, 3.0, traa=True, stage_rows=rows)
                st, got = _ao_shard(W, H, rows, it, 3.0, 3 + 2 * it)
                assert st == abi.RFX_OK and plan.ranges == got + [own] and plan.n_launches == 4 + 2 * it


def test_shard_plans_without_the_stage_are_unchanged(built):
    W, H = 640, 360
    for own in bands(H):
        for passes in (0, 2):
            for traa in (False, True):
                n = 3 + passes + traa
                plan = ShardPlan(H, 1, 0, passes, 5.0, bounds=(0, H), width=W, traa=traa)
                plan.r0, plan.r1 = own
                assert _shard(W, H, own, passes, 5.0, n) == (abi.RFX_OK, plan.ranges) and plan.n_launches == n
        for it in (0, 2):
            for traa in (False, True):
                plan = AoShardPlan(W, H, own, it, 3.0, traa=traa)
                assert _ao_shard(W, H, own, it, 3.0, plan.n_launches) == (abi.RFX_OK, plan.ranges)
