"""Reduced-resolution AO (HBAOEffect's resolutionScale) and K6's normal-texture branch on the GPU, against the oracle (which
tests/test_reference_glsl_ao.py pins to the reference's shaders): K6 on a target smaller than the depth plane, with and without a
normal plane; the Poisson pass upsampling a smaller LINEAR input (fast and exact variants); HBAOEffect end to end; C4 at 4K and
scale 0.5; and the new argument errors."""
import numpy as np
import pytest

import ao_harness as ao
import chain_harness as ch
from realism_effects_b200 import abi, effects, engine

pytestmark = pytest.mark.gpu

MAX_BAD = 1e-4  # fraction of pixels allowed outside 1e-3 relative per pass


def check(name, want, got, max_bad=MAX_BAD):
    c = ch.compare(want, got)
    print(f"{name}: bad={c['frac_bad']:.2e} max_rel_ok={c['max_rel_ok']:.1e} bit_equal={c['bit_equal']:.4f}")
    assert c["frac_bad"] <= max_bad, (name, c)
    return c


def ao_poisson_params(index: int) -> abi.PoissonParams:
    """AOEffect's denoiser pass: one plane, velocity-layout normals, LINEAR input (tests/chain_harness.ao_denoise)"""
    p = ch.poisson_params(ch.Opts(), index, False)
    p.texture_count, p.gbuffer_texture, p.input_linear = 1, 0, 1
    p.is_texture_specular[:] = [0, 0]
    p.normal_phi, p.depth_phi, p.roughness_phi, p.specular_phi = 3.25, 2.0, 0.0, 0.0
    return p


@pytest.fixture(scope="module")
def scene(built):
    return {(W, H): ch.make_inputs(W, H, 2) for W, H in ((200, 120), (201, 121))}


@pytest.mark.parametrize("size,scale", [((200, 120), 0.5), ((200, 120), 0.75), ((201, 121), 0.5)])
@pytest.mark.parametrize("with_normal", [False, True])
def test_k6_scaled_target_and_normal_plane(scene, size, scale, with_normal):
    """201 x 121 at 0.5: a 100 x 60 target with resolution (100.5, 60.5)"""
    inp = scene[size]
    f1 = inp.frames[1]
    (tw, th), res = ao.ao_target_size(*size, scale)
    normal = ao.view_normal_plane(*size, 1, f1["cam"]) if with_normal else None
    hp = ao.hbao_params(f1["cam"], 4711)
    hp.resolution[:] = list(res)
    z = np.zeros((th, tw, 4), np.float16)
    want = ao.oracle.hbao(hp, f1["depth"], inp.blue, z, out_size=(tw, th), normal=normal, resolution=res)
    ctx = engine.Context(0, inp.blue)
    try:
        out = ctx.upload(z)
        ctx.hbao(hp, ctx.upload(f1["depth"]), out, normal=None if normal is None else ctx.upload(normal))
        check(f"K6 {size} x {scale} normal={with_normal}", want, out.download())
    finally:
        ctx.close()


@pytest.mark.parametrize("fast", [True, False])
def test_poisson_upsamples_a_smaller_linear_input(scene, fast):
    inp = scene[(200, 120)]
    f1 = inp.frames[1]
    (tw, th), res = ao.ao_target_size(200, 120, 0.5)
    hp = ao.hbao_params(f1["cam"], 4711)
    small = ao.oracle.hbao(hp, f1["depth"], inp.blue, np.zeros((th, tw, 4), np.float16), out_size=(tw, th), resolution=res)
    z = np.zeros((120, 200, 4), np.float16)
    p = ao_poisson_params(1234568)
    want, _ = ao.oracle.poisson_denoise(p, f1["depth"], f1["velocity"], small, None, inp.blue, z, None)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast)
        out = ctx.upload(z)
        ctx.poisson_denoise(p, ctx.upload(f1["depth"]), ctx.upload(f1["velocity"]), ctx.upload(small), None, out, None)
        check(f"K3 from {tw}x{th} fast={fast}", want, out.download())
    finally:
        ctx.close()


class Scene:  # the host's G-buffer planes: depth, velocity (VelocityDepthNormalPass layout) and, for useNormalPass, the NormalPass output
    def __init__(self, ctx, fr, normal=None):
        self.depth, self.velocity = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"])
        self.normal = None if normal is None else ctx.upload(normal)


class Composer:
    def __init__(self, ctx, w, h):
        self.ctx, self.width, self.height = ctx, w, h
        self.inputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)
        self.outputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)


class Cam:
    def __init__(self, u):
        self.u = u

    def uniforms(self):
        return self.u


def oracle_ao_frame(inp, f1, scale, hb_index, dn_index, iterations, normal=None):
    """AOEffect.update on the oracle: K6 on the scaled target, 2 * iterations full-size Poisson passes, ao_compose of `texture`"""
    H, W = f1["depth"].shape
    (tw, th), res = ao.ao_target_size(W, H, scale)
    target = ao.oracle.hbao(ao.hbao_params(f1["cam"], hb_index.value), f1["depth"], inp.blue, np.zeros((th, tw, 4), np.float16), out_size=(tw, th),
                            normal=normal, resolution=res)
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


def test_hbao_effect_resolution_scale_normal_pass_and_no_iterations(built):
    """HBAOEffect end to end against the oracle chain, at the bar of tests/test_gpu_effects.py: resolutionScale 0.5, then 0.75
    set between frames, then iterations = 0 (the compose reads the scaled AO target); and useNormalPass with the host's normal plane"""
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
            hb = effects.HBAOEffect(comp, Cam(f1["cam"]), sc, {"blueNoiseStart": 777, "resolutionScale": 0.5, "useNormalPass": use_normal})
            bi, pbi = effects.BlueNoiseIndex(777), effects.BlueNoiseIndex(1234567)
            assert (hb.aoTarget.width, hb.aoTarget.height) == (64, 36)
            for scale, iterations in ((0.5, 1), (0.75, 1), (0.75, 0)):
                hb.resolutionScale = scale
                hb.iterations = iterations
                assert (hb.aoTarget.width, hb.aoTarget.height) == ao.ao_target_size(W, H, scale)[0]
                assert (hb.PoissonDenoisePass.texture[0].width, hb.PoissonDenoisePass.texture[0].height) == (W, H)
                hb.update(None, comp.inputBuffer)
                tex, want7 = oracle_ao_frame(inp, f1, scale, bi, pbi, iterations, normal if use_normal else None)
                assert (hb.texture is hb.aoTarget) == (iterations == 0)
                assert ch.compare(tex, hb.texture.download())["frac_bad"] <= 2e-3, (scale, iterations, use_normal)
                assert ch.compare(want7, comp.outputBuffer.download())["frac_bad"] <= 2e-3, (scale, iterations, use_normal)
            hb.dispose()
        with pytest.raises(abi.RfxError):
            effects.HBAOEffect(comp, Cam(f1["cam"]), Scene(ctx, f1), {"useNormalPass": True})  # no NormalPass output on the scene
        hb = effects.HBAOEffect(comp, Cam(f1["cam"]), Scene(ctx, f1))
        for bad in (0.0, 1.5, -0.5):
            with pytest.raises(abi.RfxError):
                hb.resolutionScale = bad
        assert hb.resolutionScale == 1 and (hb.aoTarget.width, hb.aoTarget.height) == (W, H)
        hb.dispose()
    finally:
        ctx.close()


def test_c4_4k_at_half_resolution(built):
    """C4 at 3840 x 2160 and resolutionScale 0.5: K6 on 1920 x 1080 -> 2 full-size Poisson passes -> K7 against the oracle"""
    W, H = 3840, 2160
    inp = ch.make_inputs(W, H, 1)
    fr = inp.frames[0]
    (tw, th), res = ao.ao_target_size(W, H, 0.5)
    ctx = engine.Context(0, inp.blue)
    try:
        d, v, dl = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
        hp = ao.hbao_params(fr["cam"], 778)
        hp.resolution[:] = list(res)
        zs, z = np.zeros((th, tw, 4), np.float16), np.zeros((H, W, 4), np.float16)
        want_ao = ao.oracle.hbao(hp, fr["depth"], inp.blue, zs, out_size=(tw, th), resolution=res)
        ao_g = ctx.upload(zs)
        ctx.hbao(hp, d, ao_g)
        check("C4/2 K6", want_ao, ao_g.download())
        cur, tA, tB = want_ao, z.copy(), z.copy()
        gA, gB = ctx.upload(z), ctx.upload(z)
        src_g = ao_g
        for i in range(2):
            p = ao_poisson_params(1234568 + i)
            out, _ = ao.oracle.poisson_denoise(p, fr["depth"], fr["velocity"], cur, None, inp.blue, tA if i == 0 else tB, None)
            dst_g = gA if i == 0 else gB
            ctx.poisson_denoise(p, d, v, src_g, None, dst_g, None)
            cur, src_g = out, dst_g
            check(f"C4/2 K3 pass {i}", out, dst_g.download(), max_bad=1e-3)
        want7 = ao.oracle.ao_compose(ch.ao_compose_params(), fr["depth"], cur, fr["direct"])
        outp = ctx.alloc(abi.FMT_RGBA16F, W, H)
        ctx.ao_compose(ch.ao_compose_params(), d, src_g, dl, outp)
        check("C4/2 K7", want7, outp.download(), max_bad=1e-3)
    finally:
        ctx.close()


def test_argument_errors(built):
    W, H = 64, 36
    inp = ch.make_inputs(W, H, 1)
    fr = inp.frames[0]
    ctx = engine.Context(0, inp.blue)
    try:
        d, v = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"])
        hp = ao.hbao_params(fr["cam"], 5)
        with pytest.raises(abi.RfxError, match="not larger"):
            ctx.hbao(hp, d, ctx.alloc(abi.FMT_RGBA16F, W + 1, H))
        with pytest.raises(abi.RfxError, match="RGBA8"):
            ctx.hbao(hp, d, ctx.alloc(abi.FMT_RGBA16F, W, H), normal=ctx.alloc(abi.FMT_RGBA16F, W, H))
        p = ao_poisson_params(7)
        small = ctx.alloc(abi.FMT_RGBA16F, W // 2, H // 2)
        p.input_linear = 0
        with pytest.raises(abi.RfxError, match="NEAREST"):
            ctx.poisson_denoise(p, d, v, small, None, ctx.alloc(abi.FMT_RGBA16F, W, H), None)
        p.input_linear = 1
        ctx.poisson_denoise(p, d, v, small, None, ctx.alloc(abi.FMT_RGBA16F, W, H), None)  # LINEAR: any size
        ctx.sync()
    finally:
        ctx.close()
