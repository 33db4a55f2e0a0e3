"""The passes after the SSGI chain across their option space: HBAO (K6), AO compose (K7), motion blur (K8), TRAA compose (K9), the
merged cosmetic effects (effects_kernel) and TAAPass (taa_kernel), each bit-equal to the oracle on every case of its grid.  The grids,
the branches they reach and the oracle's pinning to the reference's shaders are in tests/test_post_options_cpu.py.

Every case also checks that two launches over row ranges split at an odd row write the bytes of one launch, and for K6 that a
discarded pixel keeps the target's bytes."""
from __future__ import annotations

import numpy as np
import pytest

import orc
from realism_effects_b200 import abi
from test_post_options_cpu import (FX_CASES, K6_CASES, K7_CASES, K8_CASES, K9_SIZES, TAA_CASES, FxCase, K6Case, K7Case, K8Case, TaaCase, fx_call,
                                   inputs, k6_call, k6_oracle, k7_call, k7_oracle, k8_call, k9_call, taa_call)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    from realism_effects_b200 import engine

    c = engine.Context(0, inputs(13, 9).blue)
    yield c
    c.close()


def split_row(H: int) -> int:
    return min((H // 2) | 1, H - 1)


def bit_equal(name: str, want: np.ndarray, got: np.ndarray):
    u = np.uint8 if want.dtype == np.uint8 else np.uint16
    bad = (want.view(u) != got.view(u)).reshape(want.shape[0], want.shape[1], -1).any(-1)
    assert not bad.any(), f"{name}: {int(bad.sum())} pixels differ from the oracle, first at (y, x) = {tuple(int(v) for v in np.argwhere(bad)[0])}"


def one_and_two_launches(ctx, name: str, launch, target, H: int) -> np.ndarray:
    """launch(out, rows) over the whole frame into one copy of `target` and over [0, r) + [r, H) into another: the bytes must agree"""
    whole, split = ctx.upload(target), ctx.upload(target)
    try:
        launch(whole, (0, 0))
        r = split_row(H)
        for rows in ((0, r), (r, H)):
            launch(split, rows)
        got = whole.download()
        assert split.download().tobytes() == got.tobytes(), f"{name}: rows [0, {r}) + [{r}, {H}) differ from one launch"
        return got
    finally:
        whole.free()
        split.free()


def uploaded(ctx, *arrays):
    return [None if a is None else ctx.upload(a) for a in arrays]


def free(planes):
    for q in planes:
        if q is not None:
            q.free()


@pytest.mark.parametrize("case", K6_CASES, ids=str)
def test_k6_matches_the_oracle(ctx, case: K6Case):
    p, depth, normal, (tw, th), _, prev = k6_call(case)
    want = k6_oracle(case)
    kept = (want.view(np.uint16) == prev.view(np.uint16)).all(-1)
    assert kept.any() and not kept.all()
    ctx.set_blue_noise(inputs(case.W, case.H, case.camera).blue)
    ins = uploaded(ctx, depth, normal)
    try:
        got = one_and_two_launches(ctx, str(case), lambda out, rows: ctx.hbao(p, ins[0], out, rows=rows, normal=ins[1]), prev, th)
    finally:
        free(ins)
    assert (got.view(np.uint16)[kept] == prev.view(np.uint16)[kept]).all(), f"{case}: a discarded pixel was written"
    bit_equal(str(case), want, got)


@pytest.mark.parametrize("case", K7_CASES, ids=str)
def test_k7_matches_the_oracle(ctx, case: K7Case):
    p, depth, a, inp = k7_call(case)
    want = k7_oracle(case)
    ins = uploaded(ctx, depth, a, inp)
    try:
        got = one_and_two_launches(ctx, str(case), lambda out, rows: ctx.ao_compose(p, *ins, out, rows=rows), np.zeros_like(inp), depth.shape[0])
    finally:
        free(ins)
    bit_equal(str(case), want, got)


@pytest.mark.parametrize("case", K8_CASES, ids=str)
def test_k8_matches_the_oracle(ctx, case: K8Case):
    p, vel, inp, blue = k8_call(case)
    want = orc.motion_blur(p, vel, inp, blue)
    ctx.set_blue_noise(blue)
    ins = uploaded(ctx, vel, inp)
    try:
        got = one_and_two_launches(ctx, str(case), lambda out, rows: ctx.motion_blur(p, *ins, out, rows=rows), np.zeros_like(inp), inp.shape[0])
    finally:
        free(ins)
    bit_equal(str(case), want, got)


@pytest.mark.parametrize("size", K9_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_k9_matches_the_oracle(ctx, size):
    acc = k9_call(*size)
    want = orc.traa_compose(acc)
    ins = uploaded(ctx, acc)
    try:
        got = one_and_two_launches(ctx, f"K9 {size}", lambda out, rows: ctx.traa_compose(ins[0], out, rows=rows), np.zeros_like(acc), acc.shape[0])
    finally:
        free(ins)
    bit_equal(f"K9 {size}", want, got)


@pytest.mark.parametrize("case", FX_CASES, ids=str)
def test_effects_match_the_oracle(ctx, case: FxCase):
    p, inp, depth, vel = fx_call(case)
    want = orc.effects(p, inp, depth, vel)
    ins = uploaded(ctx, inp, depth, vel)
    try:
        got = one_and_two_launches(ctx, str(case), lambda out, rows: ctx.effects(p, *ins, out, rows=rows), np.zeros_like(inp), inp.shape[0])
    finally:
        free(ins)
    bit_equal(str(case), want, got)


@pytest.mark.parametrize("case", TAA_CASES, ids=str)
def test_taa_matches_the_oracle(ctx, case: TaaCase):
    p, inp, hist = taa_call(case)
    want = orc.taa(p, inp, hist)
    ins = uploaded(ctx, inp, hist)
    try:
        got = one_and_two_launches(ctx, str(case), lambda out, rows: ctx.taa(p, *ins, out, rows=rows), np.zeros_like(hist), inp.shape[0])
    finally:
        free(ins)
    bit_equal(str(case), want, got)


def test_taa_writes_0_for_a_negative_channel_over_history(ctx):
    """LinearTosRGB's pow(v, 0.41666) is NaN for v < 0, and mix(acc, NaN, t) clamps to 0: red -1e-4 over a history of 200 with
    cameraNotMovedFrames = 1 writes 0, not mix(200 / 255, -1e-4 * 12.92, 0.5) (which would store 100)"""
    inp = np.zeros((8, 8, 4), np.float16)
    inp[..., 0], inp[..., 3] = np.float16(-1e-4), 1.0
    hist = np.full((8, 8, 4), 200, np.uint8)
    p = abi.TaaParams()
    p.camera_not_moved_frames, p.srgb_output = 1.0, 1
    want = orc.taa(p, inp, hist)
    assert (want[..., 0] == 0).all()
    ins = uploaded(ctx, inp, hist)
    out = ctx.alloc(abi.FMT_RGBA8, 8, 8)
    try:
        ctx.taa(p, *ins, out)
        got = out.download()
    finally:
        free(ins + [out])
    assert (got[..., 0] == 0).all(), f"red {sorted(set(got[..., 0].ravel().tolist()))}"
    assert got.tobytes() == want.tobytes()
