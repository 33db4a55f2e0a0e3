"""K6h, the horizon-march AO pass, on the GPU against its CPU oracle (tests/horizon_oracle.cpp, which tests/test_horizon_ao_cpu.py holds
to an independent numpy restatement): the directions x steps grid, scaled targets, the normal plane, an orthographic camera and both
kernel variants; background texels; argument errors; C4 as the brief states it (4K, 8 x 32 -> 2 Poisson passes -> ao_compose); and
HorizonAOEffect end to end."""
import ctypes

import numpy as np
import pytest

import ao_harness as ao
import chain_harness as ch
import horizon_harness as hz
from realism_effects_b200 import abi, effects, engine
from realism_effects_b200.engine import _r
from test_gpu_ao_scale import Cam, Composer, Scene, ao_poisson_params, check

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene(built):
    s = {(W, H, False): ch.make_inputs(W, H, 2) for W, H in ((200, 120), (201, 121))}
    s[(200, 120, True)] = ch.make_inputs(200, 120, 2, orthographic=True)
    return s


def run_k6h(inp, size, scale, directions, steps, with_normal, fast, index=4711):
    f1 = inp.frames[1]
    (tw, th), res = ao.ao_target_size(*size, scale)
    normal = ao.view_normal_plane(*size, 1, f1["cam"]) if with_normal else None
    p = hz.horizon_params(f1["cam"], index, directions, steps, res)
    prev = np.full((th, tw, 4), -3.0, np.float16)
    want = hz.oracle_hbao_horizon(p, f1["depth"], inp.blue, prev, normal=normal)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast)
        out = ctx.upload(prev)
        ctx.hbao_horizon(p, ctx.upload(f1["depth"]), out, normal=None if normal is None else ctx.upload(normal))
        got = out.download()
    finally:
        ctx.close()
    assert (want[..., 3] != -3).any() and (want[..., 3] < 1).any()
    return check(f"K6h {size} x {scale} D={directions} S={steps} normal={with_normal} fast={fast}", want, got)


@pytest.mark.parametrize("fast", [True, False])
@pytest.mark.parametrize("steps", [1, 8, 32, 64])
@pytest.mark.parametrize("directions", [1, 4, 8, 32])
def test_k6h_directions_by_steps(scene, directions, steps, fast):
    run_k6h(scene[(200, 120, False)], (200, 120), 1.0, directions, steps, False, fast)


@pytest.mark.parametrize("fast", [True, False])
@pytest.mark.parametrize("with_normal", [False, True])
@pytest.mark.parametrize("size,scale", [((200, 120), 1.0), ((200, 120), 0.75), ((200, 120), 0.5), ((201, 121), 0.5)])
def test_k6h_scaled_target_and_normal_plane(scene, size, scale, with_normal, fast):
    run_k6h(scene[(*size, False)], size, scale, 8, 32, with_normal, fast)


@pytest.mark.parametrize("fast", [True, False])
@pytest.mark.parametrize("with_normal", [False, True])
def test_k6h_orthographic_camera(scene, with_normal, fast):
    run_k6h(scene[(200, 120, True)], (200, 120), 1.0, 8, 32, with_normal, fast)


def test_background_texels_keep_the_sentinel(scene):
    inp = scene[(200, 120, False)]
    f1 = inp.frames[1]
    depth = f1["depth"].copy()
    depth[:, :50] = 1.0
    prev = np.full((120, 200, 4), 12.5, np.float16)
    ctx = engine.Context(0, inp.blue)
    try:
        out = ctx.upload(prev)
        ctx.hbao_horizon(hz.horizon_params(f1["cam"], 77), ctx.upload(depth), out)
        got = out.download()
    finally:
        ctx.close()
    bg = depth == 1.0
    assert np.array_equal(got[bg].view(np.uint16), prev[bg].view(np.uint16))
    assert not (got[~bg] == np.float16(12.5)).all(-1).any()


def test_argument_errors(built):
    """every documented status of rfx_hbao_horizon_launch: 2 BAD_FORMAT, 3 SIZE_MISMATCH, 1 INVALID_ARG, 6 UNSUPPORTED (blue_noise_index 0)"""
    W, H = 64, 36
    inp = ch.make_inputs(W, H, 1)
    fr = inp.frames[0]
    ctx = engine.Context(0, inp.blue)
    try:
        d, o = ctx.upload(fr["depth"]), ctx.alloc(abi.FMT_RGBA16F, W, H)

        def status(p, depth=d, out=o, normal=None):
            return ctx.lib.rfx_hbao_horizon_launch(ctx.h, None, ctypes.byref(p), _r(depth), _r(out), _r(normal))

        ok = hz.horizon_params(fr["cam"], 5)
        assert status(ok) == 0 and status(ok, normal=ctx.alloc(abi.FMT_RGBA8, W, H)) == 0
        assert status(ok, depth=ctx.alloc(abi.FMT_RGBA32F, W, H)) == 2
        assert status(ok, out=ctx.alloc(abi.FMT_RGBA32F, W, H)) == 2
        assert status(ok, normal=ctx.alloc(abi.FMT_RGBA16F, W, H)) == 2
        assert status(ok, out=ctx.alloc(abi.FMT_RGBA16F, W + 1, H)) == 3
        assert status(ok, normal=ctx.alloc(abi.FMT_RGBA8, W // 2, H)) == 3
        for field, v in [("directions", 0), ("directions", 33), ("steps", 0), ("steps", 65), ("distance", 0.0), ("distance", -1.0),
                         ("distance", float("nan")), ("max_radius_pixels", 0.5), ("intensity", -0.1), ("angle_bias", -0.01), ("angle_bias", 1.0)]:
            p = hz.horizon_params(fr["cam"], 5)
            setattr(p, field, v)
            assert status(p) == 1, (field, v)
        p = hz.horizon_params(fr["cam"], 5)
        p.resolution[:] = [-1.0, 10.0]
        assert status(p) == 1
        assert status(hz.horizon_params(fr["cam"], 0)) == abi.ERR_UNSUPPORTED
        with pytest.raises(abi.RfxError, match="directions"):
            ctx.hbao_horizon(hz.horizon_params(fr["cam"], 5, directions=40), d, o)
        ctx.sync()
    finally:
        ctx.close()


def test_c4_literal_4k_8x32(built):
    """C4 as the brief states it: 3840 x 2160, 8 directions x 32 steps -> 2 Poisson passes -> ao_compose, against the oracle chain"""
    W, H = 3840, 2160
    inp = ch.make_inputs(W, H, 1)
    fr = inp.frames[0]
    ctx = engine.Context(0, inp.blue)
    try:
        d, v, dl = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
        p = hz.horizon_params(fr["cam"], 778, 8, 32)
        z = np.zeros((H, W, 4), np.float16)
        want_ao = hz.oracle_hbao_horizon(p, fr["depth"], inp.blue, z)
        ao_g = ctx.upload(z)
        ctx.hbao_horizon(p, d, ao_g)
        check("C4 K6h", want_ao, ao_g.download())
        cur, src_g = want_ao, ao_g
        gA, gB = ctx.upload(z), ctx.upload(z)
        for i in range(2):
            pp = ao_poisson_params(1234568 + i)
            out, _ = ao.oracle.poisson_denoise(pp, fr["depth"], fr["velocity"], cur, None, inp.blue, z, None)
            dst_g = gA if i == 0 else gB
            ctx.poisson_denoise(pp, d, v, src_g, None, dst_g, None)
            check(f"C4 K3 pass {i}", out, dst_g.download(), max_bad=1e-3)
            cur, src_g = out, dst_g
        want7 = ao.oracle.ao_compose(ch.ao_compose_params(), fr["depth"], cur, fr["direct"])
        outp = ctx.alloc(abi.FMT_RGBA16F, W, H)
        ctx.ao_compose(ch.ao_compose_params(), d, src_g, dl, outp)
        check("C4 K7", want7, outp.download(), max_bad=1e-3)
    finally:
        ctx.close()


def oracle_horizon_frame(inp, f1, scale, hb_index, dn_index, iterations, o, normal=None):
    """HorizonAOEffect.update on the oracle: K6h on the scaled target, 2 * iterations full-size Poisson passes, ao_compose"""
    H, W = f1["depth"].shape
    (tw, th), res = ao.ao_target_size(W, H, scale)
    p = hz.horizon_params(f1["cam"], hb_index.value, o["directions"], o["steps"], res, distance=o["distance"], angle_bias=o["angleBias"],
                          intensity=o["intensity"], max_radius_pixels=o["maxRadiusPixels"])
    target = hz.oracle_hbao_horizon(p, f1["depth"], inp.blue, np.zeros((th, tw, 4), np.float16), normal=normal)
    cur, tA, tB = target, np.zeros((H, W, 4), np.float16), np.zeros((H, W, 4), np.float16)
    for i in range(2 * iterations):
        out, _ = ao.oracle.poisson_denoise(ao_poisson_params(dn_index.value), f1["depth"], f1["velocity"], cur if i == 0 else tA, None, inp.blue,
                                           tA if i % 2 == 0 else tB, None)
        if i % 2 == 0:
            tA = out
        else:
            tB = out
    tex = tB if iterations > 0 else target
    return tex, ao.oracle.ao_compose(ch.ao_compose_params(), f1["depth"], tex, f1["direct"])


def test_horizon_ao_effect_end_to_end(built):
    """HorizonAOEffect against the oracle chain at tests/test_gpu_ao_scale.py's effect bar: resolutionScale 0.5, then 0.75 set between
    frames, then iterations = 0; with and without useNormalPass; a reactive option change; out-of-range options raise before a launch"""
    W, H = 128, 72
    inp = ch.make_inputs(W, H, 2)
    f1 = inp.frames[1]
    normal = ao.view_normal_plane(W, H, 1, f1["cam"])
    ctx = engine.Context(0, inp.blue)
    try:
        comp = Composer(ctx, W, H)
        comp.inputBuffer.upload(f1["direct"])
        for use_normal in (False, True):
            sc = Scene(ctx, f1, normal if use_normal else None)
            fx = effects.HorizonAOEffect(comp, Cam(f1["cam"]), sc, {"blueNoiseStart": 777, "resolutionScale": 0.5, "useNormalPass": use_normal})
            assert "spp" not in fx._options and fx.directions == 8 and fx.steps == 32
            bi, pbi = effects.BlueNoiseIndex(777), effects.BlueNoiseIndex(1234567)
            for scale, iterations, steps in ((0.5, 1, 32), (0.75, 1, 32), (0.75, 0, 32), (0.75, 1, 12)):
                fx.resolutionScale = scale
                fx.iterations = iterations
                fx.steps = steps
                assert (fx.aoTarget.width, fx.aoTarget.height) == ao.ao_target_size(W, H, scale)[0]
                fx.update(None, comp.inputBuffer)
                tex, want7 = oracle_horizon_frame(inp, f1, scale, bi, pbi, iterations, fx._options, normal if use_normal else None)
                assert (fx.texture is fx.aoTarget) == (iterations == 0)
                assert ch.compare(tex, fx.texture.download())["frac_bad"] <= 2e-3, (scale, iterations, use_normal)
                assert ch.compare(want7, comp.outputBuffer.download())["frac_bad"] <= 2e-3, (scale, iterations, use_normal)
            for k, bad in (("directions", 0), ("steps", 100), ("angleBias", 1.0), ("maxRadiusPixels", 0)):
                with pytest.raises(abi.RfxError):
                    setattr(fx, k, bad)
            assert fx.directions == 8 and fx.steps == 12
            fx.dispose()
        with pytest.raises(abi.RfxError):
            effects.HorizonAOEffect(comp, Cam(f1["cam"]), Scene(ctx, f1), {"directions": 64})
    finally:
        ctx.close()
