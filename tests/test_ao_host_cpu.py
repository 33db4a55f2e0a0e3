"""AO chain host-buffer path, host side: the rows a rank of a row-sharded group uploads (AoShardPlan.local_input_rows) against the launch
ranges of rfx_ao_shard_ranges and the kernels' own reach, and the ctypes mirror of rfx_ao_host_frame field by field.  No GPU needed."""
import ctypes as C
import math
import os
import subprocess

import pytest

from realism_effects_b200 import abi, parallel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def c_ranges(W, H, own, iterations, radius):
    n = 2 + 2 * iterations
    out = (C.c_uint32 * (2 * n))()
    assert abi.lib().rfx_ao_shard_ranges(W, H, own[0], own[1], iterations, radius, out, n) == abi.RFX_OK
    return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


def band_sets(H):
    """(bounds, rank) cases: equal bands, unequal bands (moved borders), and the first and last rank of each"""
    cases = []
    for world in (2, 3, 4):
        eq = [H * i // world for i in range(world + 1)]
        uneq = [0] + [min(H - 1, max(1, eq[i] + (-1) ** i * H // (4 * world) + 5)) for i in range(1, world)] + [H]
        for b in (eq, uneq):
            if all(b[i] < b[i + 1] for i in range(world)):
                cases += [(b, r) for r in range(world)]
    cases.append(([0, H], 0))
    return cases


@pytest.mark.parametrize("iterations", [0, 1, 2, 3])
@pytest.mark.parametrize("radius", [1.0, 3.0, 11.0, 48.0])
@pytest.mark.parametrize("size", [(640, 360), (1920, 1080), (300, 520), (96, 2048)], ids=["small", "1080p", "portrait", "tall"])
def test_local_input_rows_cover_every_launch_and_fetch(built, size, radius, iterations):
    W, H = size
    halo = math.ceil(radius * max(1.0, H / W)) + 1  # the Poisson taps' row reach, and the rows launch_gbuffer_decode widens by
    for bounds, rank in band_sets(H):
        own = (bounds[rank], bounds[rank + 1])
        plan = parallel.AoShardPlan(W, H, own, iterations, radius)
        l0, l1 = plan.local_input_rows
        assert 0 <= l0 < l1 <= H
        ranges = c_ranges(W, H, own, iterations, radius)
        assert ranges == plan.ranges
        for a, b in ranges:  # every launch: its own rows (normal at the pixel for K6, velocity at the pixel for the Poisson passes)
            assert l0 <= a and b <= l1, (own, (a, b), (l0, l1))
        for a, b in ranges[1:-1]:  # the Poisson passes: velocity at taps up to the halo, and the decode of pass 0's rows widened by it
            assert l0 <= max(0, a - halo) and min(H, b + halo) <= l1, (own, (a, b), (l0, l1))
        k7 = ranges[-1]  # K7's LINEAR fetch of `input` at the pixel centre touches row y +- 1
        assert k7 == own and l0 <= max(0, k7[0] - 1) and min(H, k7[1] + 1) <= l1
        if iterations == 0:  # no Poisson pass: nothing reads beyond K6's rows
            assert (l0, l1) == ranges[0]


def test_local_input_rows_of_one_rank_is_the_frame(built):
    for iterations in (0, 2):
        assert parallel.AoShardPlan(640, 360, (0, 360), iterations, 3.0).local_input_rows == (0, 360)


def test_ctypes_mirror_of_the_host_frame_matches_c(tmp_path):
    fields = [f[0] for f in abi.AoHostFrame._fields_]
    body = f'printf("sizeof %zu\\n", sizeof(rfx_ao_host_frame));'
    body += "".join(f'printf("{n} %zu\\n", offsetof(rfx_ao_host_frame, {n}));' for n in fields)
    src = tmp_path / "off.cpp"
    src.write_text(f'#include <cstddef>\n#include <cstdio>\n#include "rfx.h"\nint main(){{{body} return 0;}}\n')
    exe = tmp_path / "off"
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = {k: int(v) for k, v in (l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())}
    assert out.pop("sizeof") == C.sizeof(abi.AoHostFrame)
    assert out == {n: getattr(abi.AoHostFrame, n).offset for n in fields}
    hdr = open(os.path.join(ROOT, "include", "rfx.h")).read()
    decl = hdr[hdr.index("typedef struct rfx_ao_host_frame {"):hdr.index("} rfx_ao_host_frame;")]
    for n in fields:  # every member the header declares is mirrored (the offsets above fail to compile for a member it lacks)
        assert n in decl
