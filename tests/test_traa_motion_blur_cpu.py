"""TRAAEffect + MotionBlurEffect as one EffectPass (rfx_traa_motion_blur_launch), on the CPU: the oracle (tests/mb_oracle.cpp) against the
reference's own shaders (tests/mb_harness.reference, where they can run) and against their recorded digests (tests/golden/
reference_pins_mb.json) over K8's option space: samples 1 / 16 / 32, intensity 0.25 / 1 / 3, jitter 0 / 1, frame 0 (the tiled blue-noise
lookup) and non-zero, deltaTime clamped at 1/1000 and large, still pixels and taps clamped at the frame's edges.  Plus the C-ABI mirrors
of the new entry points."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest

import mb_harness as mb
import orc
from realism_effects_b200 import abi
from test_post_options_cpu import K8Case, color_plane, k8_call

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MB_CASES = [
    K8Case(),
    K8Case(203, 117, samples=1, intensity=0.25, jitter=0.0, frame=0),
    K8Case(200, 120, samples=32, intensity=3.0, dt=1e-4, resolution=(150.5, 90.25), vmax=0.2),
    K8Case(90, 160, samples=32, jitter=0.0, frame=0, blue=96),
    K8Case(3840, 16, samples=16, intensity=0.25, frame=3),
    K8Case(13, 9, samples=1, dt=1e-4, resolution=(26.0, 18.0)),
    K8Case(203, 117, samples=16, intensity=3.0, dt=0.5, frame=0, vmax=0.2),
]


def mb_call(case: K8Case):
    """(params, velocity, accumulated, input buffer, blue noise): K8's inputs, and an accumulated plane unlike the input buffer"""
    p, vel, inp, blue = k8_call(case)
    acc = color_plane(case.H, case.W, 8101, 4.0)
    return p, vel, acc, inp, blue


def tap_span(p: abi.MotionBlurParams, vel: np.ndarray):
    """per pixel: whether it moves, and its start / end uv before the clamp (float64, as motion_blur.frag forms them up to rounding)"""
    H, W = vel.shape[:2]
    v = vel[..., :2].astype(np.float64)
    moved = (v * v).sum(-1) > 1e-9
    ys, xs = np.meshgrid((np.arange(H) + 0.5) / H, (np.arange(W) + 0.5) / W, indexing="ij")
    uv = np.stack([xs, ys], -1)
    half = v * float(p.intensity) * 0.5 * (0.01 / float(p.delta_time))
    jit = np.abs(v * float(p.intensity) * float(p.jitter) * (0.01 / float(p.delta_time)))  # |jitterOffset| * frameSpeed at most
    return moved, uv - half - jit, uv + half + jit


def test_grid_reaches_every_configuration():
    assert {c.samples for c in MB_CASES} == {1, 16, 32} and {c.intensity for c in MB_CASES} == {0.25, 1.0, 3.0}
    assert {c.jitter for c in MB_CASES} == {0.0, 1.0} and {c.frame == 0 for c in MB_CASES} == {True, False}
    dts = [max(1 / 1000, c.dt) for c in MB_CASES]
    assert min(dts) == 1 / 1000 and max(dts) >= 0.1
    still = clamped = 0
    for c in MB_CASES:
        p, vel, *_ = mb_call(c)
        moved, lo, hi = tap_span(p, vel)
        still += int((~moved).sum())
        clamped += int((moved & ((lo < 0).any(-1) | (hi > 1).any(-1))).sum())
    assert still > 0 and clamped > 0


@pytest.mark.parametrize("case", MB_CASES, ids=str)
def test_oracle_equals_the_reference_pins(case):
    want = mb.pins()
    assert str(case) in want, f"{case}: no recorded digest (mint with tests/golden/make_golden_mb.py)"
    assert mb.digest(mb.oracle(*mb_call(case))) == want[str(case)]


@pytest.mark.parametrize("case", MB_CASES, ids=str)
def test_oracle_equals_the_reference_shaders(case):
    if not mb.reference_available(case.samples):
        pytest.skip("the reference's shaders are neither buildable nor prebuilt here (the pins above hold the comparison)")
    args = mb_call(case)
    got, want = mb.oracle(*args), mb.reference(*args)
    assert got.view(np.uint16).tobytes() == want.view(np.uint16).tobytes()


def test_the_taps_read_the_input_buffer_and_still_pixels_show_traa():
    """The merged pass is not K8 over K9's output: a moving pixel's taps read the frame before TRAA.  A still pixel writes K9's texel."""
    p, vel, acc, inp, blue = mb_call(MB_CASES[0])
    got = mb.oracle(p, vel, acc, inp, blue).view(np.uint16)
    k9 = orc.traa_compose(acc).view(np.uint16)
    chained = orc.motion_blur(p, vel, k9.view(np.float16), blue).view(np.uint16)
    moved, *_ = tap_span(p, vel)
    assert (~moved).any() and np.array_equal(got[~moved], k9[~moved])
    assert (got[moved] != chained[moved]).any(axis=-1).mean() > 0.5


def test_ctypes_mirrors_of_the_new_entry_points(built):
    hdr = open(os.path.join(ROOT, "include", "rfx.h")).read()
    lib = abi.lib()
    for name in ("rfx_traa_motion_blur_launch", "rfx_ssgi_chain_set_motion_blur", "rfx_ao_chain_set_motion_blur"):
        m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", hdr)
        assert m and name in abi.EXPORTS
        assert len(getattr(lib, name).argtypes) == len(m.group(1).split(",")), name
    assert lib.rfx_traa_motion_blur_launch.argtypes[2] == lib.rfx_motion_blur_launch.argtypes[2]  # rfx_motion_blur_params, unchanged
