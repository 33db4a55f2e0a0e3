"""GPU tests of the plugin-surface mirror (realism_effects_b200/effects.py): the classes a reference user instantiates
(SSGIEffect / TRAAEffect / MotionBlurEffect / HBAOEffect / VelocityDepthNormalPass) produce what the oracle produces
when driven like the reference's frame loop."""
import numpy as np
import pytest

import chain_harness as ch
from realism_effects_b200 import abi, effects, engine, synth

pytestmark = pytest.mark.gpu


class Scene:  # what stands in for the rasterised G-buffer / velocity render targets
    def __init__(self, ctx):
        self.ctx = ctx
        self.depth = self.gbuffer = self.velocity = None

    def load(self, fr):
        for p in (self.depth, self.gbuffer, self.velocity):
            if p is not None:
                p.free()
        self.depth, self.gbuffer, self.velocity = self.ctx.upload(fr["depth"]), self.ctx.upload(fr["gbuffer"]), self.ctx.upload(fr["velocity"])


class Composer:
    def __init__(self, ctx, w, h):
        self.ctx, self.width, self.height = ctx, w, h
        self.inputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)
        self.outputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)


class Cam:
    def __init__(self):
        self.u = None

    def uniforms(self):
        return self.u


def test_ssgi_effect_matches_oracle_chain(built):
    import orc

    inp = ch.make_inputs(160, 90, 3)
    o = ch.Opts()
    ref = ch.run_oracle_chain(inp, o)
    ctx = engine.Context(0, inp.blue)
    try:
        scene, comp, cam = Scene(ctx), Composer(ctx, 160, 90), Cam()
        cam.u = inp.frames[0]["cam"]
        fx = effects.SSGIEffect(comp, scene, cam, {"blueNoiseStart": o.blue_noise_start})
        assert fx.steps == 20 and fx.refineSteps == 5 and fx.denoiseIterations == 1 and effects.SSGIEffect.DefaultOptions["normalPhi"] == 50
        fx.setEnvironment(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        for t, fr in enumerate(inp.frames):
            scene.load(fr)
            comp.inputBuffer.upload(fr["direct"])
            cam.u = fr["cam"]
            fx.update(None, comp.inputBuffer)
            got = fx._chain.download(0)
            c = ch.compare(ref[t]["composed"], got)
            assert c["frac_bad"] <= 6e-3 and ch.compare(ref[t]["composed"], got, rtol=4e-3)["frac_bad"] <= 1.5e-3, (t, c)
            want5 = orc.ssgi_compose(fr["depth"], got, fr["direct"])  # K5 on the engine's own GI plane
            assert ch.compare(want5, comp.outputBuffer.download())["n_bad"] == 0
        # reactive option: the setter reconfigures the native chain and resets the history (SSGIEffect.js:203-209)
        fx.steps = 8
        assert fx.steps == 8 and fx._chain.opt.steps == 8
        fx.update(None, comp.inputBuffer)
        tr_alpha = fx._chain.download(2)[..., 3]
        assert tr_alpha.max() == 0.0  # keepData = 0 => no accumulated history on the frame after a reset
        fx.dispose()
    finally:
        ctx.close()


def test_hbao_effect_traa_effect_motion_blur_effect(built):
    import orc

    inp = ch.make_inputs(128, 72, 2)
    f0, f1 = inp.frames
    W, H = 128, 72
    ctx = engine.Context(0, inp.blue)
    try:
        scene, comp, cam = Scene(ctx), Composer(ctx, W, H), Cam()
        scene.load(f1)
        cam.u = f1["cam"]
        comp.inputBuffer.upload(f1["direct"])
        # ---- HBAOEffect: K6 -> 2 Poisson passes (1 plane, velocity-layout normals) -> K7
        hb = effects.HBAOEffect(comp, cam, scene, {"blueNoiseStart": 777})
        assert hb.spp == 8 and hb.distance == 2 and hb.bias == 40 and hb.power == 2
        hb.update(None, comp.inputBuffer)
        bi = effects.BlueNoiseIndex(777)
        z = np.zeros((H, W, 4), np.float16)
        ao = orc.hbao(ch.hbao_params(f1["cam"], bi.value), f1["depth"], inp.blue, z)
        pbi = effects.BlueNoiseIndex(1234567)
        cur, tgtA, tgtB = ao, z.copy(), z.copy()
        for i in range(2):
            p = ch.poisson_params(ch.Opts(), pbi.value, False)
            p.texture_count, p.gbuffer_texture, p.input_linear = 1, 0, 1
            p.is_texture_specular[:] = [0, 0]
            p.normal_phi, p.depth_phi, p.roughness_phi, p.specular_phi = 3.25, 2.0, 0.0, 0.0
            src = cur if i == 0 else tgtA
            out, _ = orc.poisson_denoise(p, f1["depth"], f1["velocity"], src, None, inp.blue, tgtA if i == 0 else tgtB, None)
            if i == 0:
                tgtA = out
            else:
                tgtB = out
        assert ch.compare(tgtB, hb.texture.download())["frac_bad"] <= 2e-3
        want7 = orc.ao_compose(ch.ao_compose_params(), f1["depth"], hb.texture.download(), f1["direct"])
        assert ch.compare(want7, comp.outputBuffer.download())["frac_bad"] <= 2e-3
        hb.dispose()
        # ---- TRAAEffect: frame 0 seeds the history, frame 1 reprojects it
        vdn = effects.VelocityDepthNormalPass(scene, cam)
        traa = effects.TRAAEffect(scene, cam, vdn)
        assert traa.options["maxBlend"] == 0.9 and traa.options["confidencePower"] == 4 and traa.options["logTransform"] is True
        scene.load(f0)
        cam.u = f0["cam"]
        comp.inputBuffer.upload(f0["direct"])
        traa.update(None, comp.inputBuffer)
        hist = traa.temporalReprojectPass.accumulated.download()
        scene.load(f1)
        cam.u = f1["cam"]
        comp.inputBuffer.upload(f1["direct"])
        traa.update(None, comp.inputBuffer)
        p = ch.traa_temporal_params(abi.make_camera(f1["cam"]), f1["cam"]["position"], f0["cam"], 1.0)
        want, _ = orc.temporal_reproject(p, f1["direct"], f1["velocity"], hist, None, z, None, out_half=True)
        assert ch.compare(want, traa.temporalReprojectPass.accumulated.download())["frac_bad"] <= 2e-3
        traa.compose(comp.outputBuffer)
        assert (comp.outputBuffer.download()[..., 3] == 1).all()
        traa.dispose()
        # ---- MotionBlurEffect
        mb = effects.MotionBlurEffect(vdn)
        assert (mb.intensity, mb.jitter, mb.samples) == (1, 1, 16)
        vel = ch.rotation_velocity_field(W, H, f1["depth"])
        scene.velocity.upload(vel)
        mb._frame = 7
        mb.update(None, comp.inputBuffer, 1 / 60, comp.outputBuffer)
        want = orc.motion_blur(ch.motion_blur_params(W, H, frame=7), vel, f1["direct"], inp.blue)
        assert ch.compare(want, comp.outputBuffer.download())["frac_bad"] <= 2e-3
    finally:
        ctx.close()


@pytest.mark.parametrize("flip_y,size", [pytest.param(f, (w, h), id=str(f) if (w, h) == (256, 128) else f"{f}-{w}x{h}")
                                         for w, h in ((256, 128), (100, 50), (37, 19)) for f in (False, True)])
def test_env_cdf_tables_built_on_device_are_bit_identical(built, flip_y, size):
    """rfx_env_build (SURVEY.md §8f row 1): the device-built marginal / conditional inverse-CDF tables and totalSum equal the
    restatement of `gatherData` (EquirectHdrInfoUniform.js:149-245, synth.build_env_cdf) bit for bit, including the reference's
    mirroring "un-flip" for flipY textures (A4); and K1 gives the same bytes with either set of tables.  Odd sizes: the flipY mirror
    has a middle row, and the env map's mip chain has levels of odd size (K1's trilinear fetches)."""
    w, h = size
    env = synth.synthetic_env(w, h)
    env[h * 40 // 128:h * 60 // 128, w * 100 // 256:w * 140 // 256, :3] = 0  # a black patch: flat CDF stretches (ties in the binary search)
    env[h * 7 // 128] = 0                                                    # an all-black row: cumulativeRowWeight == 0 branch
    marg, cond, total = synth.build_env_cdf(env.astype(np.float32), flip_y=flip_y)
    inp = ch.make_inputs(96, 54, 1)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.build_env(env, flip_y=flip_y)
        gm, gc, gt = ctx.env_tables()
        assert gt == total
        assert np.array_equal(gm.view(np.uint32), marg.view(np.uint32))
        assert np.array_equal(gc.view(np.uint32), cond.view(np.uint32))
        fr = inp.frames[0]
        p = ch.ssgi_params(ch.Opts(), abi.make_camera(fr["cam"]), 4242, (w, h))
        planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "direct")]
        out_dev = ctx.alloc(abi.FMT_RGBA32F, 96, 54)
        ctx.ssgi_trace(p, planes[0], planes[1], None, planes[2], None, out_dev)
        a = out_dev.download()
        ctx.set_env(env, marg, cond, total)
        ctx.ssgi_trace(p, planes[0], planes[1], None, planes[2], None, out_dev)
        assert a.tobytes() == out_dev.download().tobytes()
    finally:
        ctx.close()


@pytest.mark.parametrize("exp2", [False, True])
def test_ssgi_compose_fog_and_debug(built, exp2):
    """K5 with scene fog (three.js Fog / FogExp2 through <fog_fragment> on vFogDepth = -getViewZ(depth) * 0.4, SSGIEffect.js:34-43,
    404-412) and the isDebug pass-through, against the oracle."""
    import orc

    inp = ch.make_inputs(128, 72, 1)
    fr = inp.frames[0]
    rng = np.random.default_rng(3)
    gi = rng.uniform(0, 2, (72, 128, 4)).astype(np.float32)
    p = abi.SsgiComposeParams()
    p.use_fog, p.fog_exp2, p.perspective = 1, int(exp2), 1
    p.fog_color[:] = [0.6, 0.7, 0.8]
    p.fog_near, p.fog_far, p.fog_density = 2.0, 30.0, 0.05
    p.camera_near, p.camera_far = float(fr["cam"]["near"]), float(fr["cam"]["far"])
    ctx = engine.Context(0, inp.blue)
    try:
        d, g, sc = ctx.upload(fr["depth"]), ctx.upload(gi), ctx.upload(fr["direct"])
        out = ctx.alloc(abi.FMT_RGBA16F, 128, 72)
        ctx.ssgi_compose(d, g, sc, out, params=p)
        want = orc.ssgi_compose(fr["depth"], gi, fr["direct"], p)
        nofog = orc.ssgi_compose(fr["depth"], gi, fr["direct"])
        assert ch.compare(want, out.download())["n_bad"] == 0
        assert not np.array_equal(want, nofog)                                         # the fog does something on foreground pixels ...
        bg = fr["depth"] == 1.0
        assert np.array_equal(want[bg], nofog[bg])                                     # ... and nothing on the background (scene colour)
        p.is_debug = 1
        ctx.ssgi_compose(d, g, sc, out, params=p)
        assert np.array_equal(out.download(), gi.astype(np.float16))                   # isDebug: the GI texture passes through
    finally:
        ctx.close()


def test_gbuffer_ingest_is_bit_identical_to_the_oracle_and_feeds_the_chain(built):
    """rfx_gbuffer_ingest_launch (SURVEY.md §8f row 2): every input-format combination against orc_gbuffer_ingest bit for bit, row-block
    launches, and the ingested planes driving K1 give the bytes the generator's own packed planes give."""
    import orc

    W, H = 200, 120
    fr = synth.render_frame(W, H, 1)
    s = {k: v.cpu().numpy() for k, v in fr.soa.items()}
    d = fr.depth.numpy()
    variants = [
        dict(albedo=s["albedo"], normal=s["normal"], material=s["material"], emissive=s["emissive"], motion=s["motion"], kw=dict(normalize_normals=False)),
        dict(albedo=(s["albedo"].astype(np.float32) / 255).astype(np.float16), normal=s["normal"].astype(np.float16),
             material=(s["material"].astype(np.float32) * 255).round().astype(np.uint8), emissive=s["emissive"], motion=s["motion"].astype(np.float16),
             kw=dict(motion_scale=(0.5, 2.0))),
        dict(albedo=s["albedo"], normal=s["normal"].astype(np.float16), material=s["material"], emissive=None, motion=None, kw={}),
    ]
    ctx = engine.Context(0, synth.load_blue_noise())
    try:
        dd = ctx.upload(d)
        for v in variants:
            want_g, want_v = orc.gbuffer_ingest(v["albedo"], v["normal"], v["material"], v["emissive"], v["motion"], d, **v["kw"])
            up = lambda a: None if a is None else ctx.upload(a)  # noqa: E731
            planes = [up(v[k]) for k in ("albedo", "normal", "material", "emissive", "motion")]
            og, ov = ctx.alloc(abi.FMT_RGBA32F, W, H), ctx.alloc(abi.FMT_RGBA32F, W, H)
            ctx.gbuffer_ingest(*planes, dd, og, ov, **v["kw"])
            assert og.download().view(np.uint32).tobytes() == want_g.view(np.uint32).tobytes()
            assert ov.download().view(np.uint32).tobytes() == want_v.view(np.uint32).tobytes()
            og2, ov2 = ctx.alloc(abi.FMT_RGBA32F, W, H), ctx.alloc(abi.FMT_RGBA32F, W, H)
            for r in ((0, 37), (37, H)):
                ctx.gbuffer_ingest(*planes, dd, og2, ov2, rows=r, **v["kw"])
            assert og2.download().tobytes() == og.download().tobytes() and ov2.download().tobytes() == ov.download().tobytes()
        # variant 0 reproduces the generator's velocity plane and the diffuse / normal words of its gBuffer; K1 on the ingested planes
        v = variants[0]
        planes = [ctx.upload(v[k]) for k in ("albedo", "normal", "material", "emissive", "motion")]
        og, ov = ctx.alloc(abi.FMT_RGBA32F, W, H), ctx.alloc(abi.FMT_RGBA32F, W, H)
        ctx.gbuffer_ingest(*planes, dd, og, ov, normalize_normals=False)
        assert ov.download().tobytes() == fr.velocity.numpy().tobytes()
        with pytest.raises(abi.RfxError):
            ctx.gbuffer_ingest(planes[1], planes[1], planes[2], None, None, dd, og, ov)   # an RGBA32F albedo is rejected (BAD_FORMAT)
    finally:
        ctx.close()


def test_cosmetic_effects_tail_kernel_and_taa(built):
    """rfx_effects_launch (Sharpness / LensDistortion / GradualBackground / Sparkle merged like an EffectPass) and rfx_taa_launch, bit-equal to
    the oracle (which equals the reference's shaders bit for bit, tests/test_reference_glsl.py); row-block launches are exact."""
    import orc

    W, H = 200, 120
    inp = ch.make_inputs(W, H, 2)
    f1 = inp.frames[1]
    ctx = engine.Context(0, inp.blue)
    try:
        src, d, v = ctx.upload(f1["direct"]), ctx.upload(f1["depth"]), ctx.upload(f1["velocity"])
        for effs, sp in ch.FX_CASES:
            p = ch.fx_params(f1["cam"], effs, sp)
            want = orc.effects(p, f1["direct"], f1["depth"], f1["velocity"])
            out = ctx.alloc(abi.FMT_RGBA16F, W, H)
            ctx.effects(p, src, d, v, out)
            got = out.download()
            assert got.view(np.uint16).tobytes() == want.view(np.uint16).tobytes(), (effs, sp, ch.compare(want, got))
            parts = ctx.alloc(abi.FMT_RGBA16F, W, H)
            ctx.effects(p, src, d, v, parts, rows=(0, 41))
            ctx.effects(p, src, d, v, parts, rows=(41, H))
            assert parts.download().tobytes() == got.tobytes()
        hist = np.random.default_rng(1).integers(0, 256, (H, W, 4), dtype=np.uint8)
        hd = ctx.upload(hist)
        for p in ch.taa_cases():
            out = ctx.alloc(abi.FMT_RGBA8, W, H)
            ctx.taa(p, src, hd, out)
            want = orc.taa(p, f1["direct"], hist)
            got = out.download()
            assert np.array_equal(got, want), (p.camera_not_moved_frames, p.srgb_output, int((got != want).sum()))
        with pytest.raises(abi.RfxError):
            ctx.effects(ch.fx_params(f1["cam"], [abi.FX_SPARKLE]), src, d, None, ctx.alloc(abi.FMT_RGBA16F, W, H))  # Sparkle without the velocity plane
    finally:
        ctx.close()


def test_effect_pass_and_taa_pass_host_classes(built):
    """effects.EffectPass(camera, SharpnessEffect, GradualBackgroundEffect, SparkleEffect) = one merged launch; effects.TAAPass accumulates while the
    camera stands still (cameraNotMovedFrames 0, 1, 2 ...) and restarts when it moves."""
    import orc

    W, H = 128, 72
    inp = ch.make_inputs(W, H, 2)
    f1 = inp.frames[1]
    ctx = engine.Context(0, inp.blue)
    try:
        scene, comp, cam = Scene(ctx), Composer(ctx, W, H), Cam()
        scene.load(f1)
        cam.u = f1["cam"]
        comp.inputBuffer.upload(f1["direct"])
        vdn = effects.VelocityDepthNormalPass(scene, cam)
        sharp, grad, spark = effects.SharpnessEffect({"sharpness": 1.5}), effects.GradualBackgroundEffect(cam, scene.depth, (0.2, 0.3, 0.5), 20.5), effects.SparkleEffect(cam, vdn)
        assert effects.SharpnessEffect().sharpness == 1 and effects.LensDistortionEffect().alphax == -0.05 and spark.spread == 1
        effects.EffectPass(cam, sharp, grad, spark).render(None, comp.inputBuffer, comp.outputBuffer)
        want = orc.effects(ch.fx_params(f1["cam"], [abi.FX_SHARPNESS, abi.FX_GRADUAL_BACKGROUND, abi.FX_SPARKLE]), f1["direct"], f1["depth"], f1["velocity"])
        assert ch.compare(want, comp.outputBuffer.download())["frac_bad"] <= 1e-4
        taa = effects.TAAPass(cam)
        taa.setSize(W, H, ctx)
        hist = np.zeros((H, W, 4), np.uint8)
        for n_expected in (0, 1, 2):
            shown = taa.render(None, comp.inputBuffer).download()
            assert taa.cameraNotMovedFrames == n_expected
            p = abi.TaaParams()
            p.camera_not_moved_frames, p.srgb_output = float(n_expected), 1
            want = orc.taa(p, f1["direct"], hist)
            assert np.abs(shown.astype(np.int32) - want.astype(np.int32)).max() <= 1
            hist = shown
        cam.u = inp.frames[0]["cam"]
        taa.render(None, comp.inputBuffer)
        assert taa.cameraNotMovedFrames == 0
        taa.dispose()
    finally:
        ctx.close()
