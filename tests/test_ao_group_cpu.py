"""Row-sharded AO chain, host side: rfx_ao_shard_ranges against its Python mirror parallel.AoShardPlan, the containment of every row a
later launch reads in the earlier launch's range (enumerated from the Poisson tap table), the argument checks, and the ctypes mirrors of
the new structs.  No GPU needed."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from realism_effects_b200 import abi, parallel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SQ = 1.41421356237
POISSON = [(-1.0, 0.0), (0.0, -1.0), (1.0, 0.0), (0.0, 1.0), (-0.25 * SQ, -0.25 * SQ), (0.25 * SQ, -0.25 * SQ), (0.25 * SQ, 0.25 * SQ),
           (-0.25 * SQ, 0.25 * SQ)]  # poisson_denoise.frag's tap table (k_denoise.cu)


def c_ranges(W, H, own, iterations, radius):
    n = 2 + 2 * iterations
    out = (C.c_uint32 * (2 * n))()
    st = abi.lib().rfx_ao_shard_ranges(W, H, own[0], own[1], iterations, radius, out, n)
    assert st == abi.RFX_OK
    return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


def bands(H, n, shift=0):
    b = [int(round(H * i / n / 16.0)) * 16 for i in range(n)] + [H]
    return [0] + [x + shift for x in b[1:-1]] + [H]


@pytest.mark.parametrize("iterations", [0, 1, 2, 3])
@pytest.mark.parametrize("radius", [3.0, 11.0, 32.0])
@pytest.mark.parametrize("size", [(640, 360), (300, 520)], ids=["landscape", "portrait"])
def test_c_ranges_equal_the_python_plan(built, iterations, radius, size):
    W, H = size
    for n in range(2, 9):
        for shift in (0, 16, -16, 5):
            b = bands(H, n, shift)
            for r in range(n):
                own = (b[r], b[r + 1])
                plan = parallel.AoShardPlan(W, H, own, iterations, radius)
                got = c_ranges(W, H, own, iterations, radius)
                assert got == plan.ranges, (size, n, shift, r)
                assert got[-1] == own
                for (a0, a1), (b0, b1) in zip(got, got[1:]):  # every launch covers the next one's rows
                    assert a0 <= b0 and b1 <= a1


def _rows_read(W, H, rows, radius, k7):
    """rows a launch over output rows `rows` reads of its input plane: K7's LINEAR fetch at the pixel centre, or every Poisson tap at
    every rotation of the blue-noise table and flatness in [0.25, 1] with its LINEAR footprint (a quad's helper pixel outside the range
    takes its derivatives from the input planes and returns before any tap)"""
    y = np.arange(rows[0], rows[1], dtype=np.float64)
    if k7:
        yy = (y + 0.5) - 0.5  # clamp-to-edge: rows outside the frame read its first / last row
        return max(0, int(np.floor(yy).min())), min(H - 1, int(np.floor(yy).max()) + 1)
    lo, hi = math.inf, -math.inf
    ang = np.arange(256) / 255.0 * 2.0 * math.pi
    s, c = np.sin(ang), np.cos(ang)
    for flat in (0.25, 1.0):
        k = radius * flat
        for px, py in POISSON:
            ox, oy = px / W, py / H
            dv = (k * -s) * ox + (k * c) * oy  # m01 * ox + m11 * oy, as the kernel rotates
            for yq in (y.min(), y.max()):
                v = (yq + 0.5) / H + dv
                t = v * H - 0.5
                lo, hi = min(lo, math.floor(t.min())), max(hi, math.floor(t.max()) + 1)
    return max(0, int(lo)), min(H - 1, int(hi))


@pytest.mark.parametrize("iterations", [0, 1, 2])
@pytest.mark.parametrize("size,radius", [((640, 360), 3.0), ((300, 520), 11.0), ((640, 360), 32.0)])
def test_every_row_a_launch_reads_lies_in_the_earlier_launch_range(built, iterations, size, radius):
    W, H = size
    b = bands(H, 4, 16)
    for r in range(4):
        own = (b[r], b[r + 1])
        rng = c_ranges(W, H, own, iterations, radius)
        for k in range(1, len(rng)):
            lo, hi = _rows_read(W, H, rng[k], radius, k7=(k == len(rng) - 1))
            assert rng[k - 1][0] <= lo and hi < rng[k - 1][1], (size, iterations, r, k, (lo, hi), rng[k - 1])


def test_bad_arguments_are_rejected(built):
    lib = abi.lib()
    out = (C.c_uint32 * 8)()
    bad = [
        (64, 128, 0, 64, 1, 3.0, out, 3),       # n_launches != 2 + 2 * iterations
        (64, 128, 0, 64, -1, 3.0, out, 0),      # iterations < 0
        (64, 128, 64, 64, 1, 3.0, out, 4),      # empty band
        (64, 128, 0, 129, 1, 3.0, out, 4),      # band beyond the frame
        (0, 128, 0, 64, 1, 3.0, out, 4),        # width 0
        (64, 128, 0, 64, 1, float("nan"), out, 4),
        (64, 128, 0, 64, 1, float("inf"), out, 4),
        (64, 128, 0, 64, 1, 3.0, None, 4),
    ]
    for a in bad:
        assert lib.rfx_ao_shard_ranges(*a) == 1, a


def test_ctypes_mirrors_of_the_ao_structs_match_c(tmp_path):
    names = {"rfx_ao_chain_options": abi.AoChainOptions, "rfx_ao_frame": abi.AoFrame}
    src = tmp_path / "sz.c"
    body = "\n".join(f'printf("{n} %zu\\n", sizeof({n}));' for n in names)
    body += '\nprintf("opt_color %zu\\n", offsetof(rfx_ao_chain_options, color));\nprintf("frame_depth %zu\\n", offsetof(rfx_ao_frame, depth));'
    src.write_text(f'#include <stddef.h>\n#include <stdio.h>\n#include "rfx.h"\nint main(void){{{body} return 0;}}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for n, cls in names.items():
        assert int(out[n]) == C.sizeof(cls), (n, out[n], C.sizeof(cls))
    assert int(out["opt_color"]) == abi.AoChainOptions.color.offset
    assert int(out["frame_depth"]) == abi.AoFrame.depth.offset


def test_options_from_the_effect_tables():
    from realism_effects_b200 import effects, engine

    o = engine.ao_chain_options(640, 360, {"blueNoiseStart": 777, "iterations": 2})
    assert (o.algorithm, o.spp, o.iterations, o.blue_noise_start, o.denoise_blue_noise_start) == (abi.AO_HBAO, 8, 2, 777, 1234567)
    assert o.normal_phi == pytest.approx(effects.defaultAOOptions["normalPhi"])
    h = engine.ao_chain_options(640, 360, {"directions": 4}, horizon=True)
    assert (h.algorithm, h.directions, h.steps) == (abi.AO_HORIZON, 4, 32)
    with pytest.raises(abi.RfxError):
        engine.ao_chain_options(640, 360, {"directions": 0}, horizon=True)
