"""GPU tests of the debug views (SSGIEffect's `outputTexture`, src/ssgi/SSGIEffect.js:228-251): gbuffer_debug_kernel and K5's debug
branch against the oracle of tests/debug_oracle.cpp (pinned to the reference's shaders by tests/test_debug_views_cpu.py), SSGIEffect /
SSREffect switching views between frames, the chain's TRAA tail with a view, and the refusals of a view in a row-sharded group."""
import ctypes as C

import numpy as np
import pytest

import chain_harness as ch
import debug_views as D
from realism_effects_b200 import abi, effects, engine

pytestmark = pytest.mark.gpu


def _same(a, b):
    """bit-equal, except that two NaNs of any payload are equal (a packed G-buffer texel can be a NaN pattern; fp16 NaN payloads differ)"""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype
    bits = a.view(np.uint16 if a.dtype == np.float16 else np.uint32) == b.view(np.uint16 if b.dtype == np.float16 else np.uint32)
    return bool((bits | (np.isnan(a) & np.isnan(b))).all())


@pytest.mark.parametrize("size", [(200, 120), (203, 117), (3840, 2160)])
def test_gbuffer_debug_kernel_matches_oracle_every_mode(built, size):
    W, H = size
    g = D.debug_frame(W, H)["gbuffer"]
    ctx = engine.Context(0)
    try:
        gb, out = ctx.upload(g), ctx.alloc(abi.FMT_RGBA32F, W, H)
        for mode in (*range(6), -1, 9):
            out.clear()
            ctx.gbuffer_debug(mode, gb, out)
            assert out.download().tobytes() == D.oracle.gbuffer_debug(mode, g).tobytes(), mode
        # row ranges: two launches over [0, H/3) and [H/3, H) write the bytes of one
        out.clear()
        ctx.gbuffer_debug(2, gb, out, rows=(0, H // 3))
        ctx.gbuffer_debug(2, gb, out, rows=(H // 3, H))
        assert out.download().tobytes() == D.oracle.gbuffer_debug(2, g).tobytes()
    finally:
        ctx.close()


def test_gbuffer_debug_emissive_every_exponent(built):
    """decodeRGBE8<true> against the oracle's exp2cr for all 256 exponent bytes (the only values fExp takes), bit for bit"""
    g = D.rgbe_gbuffer()
    ctx = engine.Context(0)
    try:
        out = ctx.alloc(abi.FMT_RGBA32F, g.shape[1], g.shape[0])
        ctx.gbuffer_debug(5, ctx.upload(g), out)
        assert out.download().tobytes() == D.oracle.gbuffer_debug(5, g).tobytes()
    finally:
        ctx.close()


@pytest.mark.parametrize("size", [(200, 120), (203, 117)])
def test_k5_debug_matches_oracle_every_source(built, size):
    W, H = size
    ctx = engine.Context(0)
    try:
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        p = abi.SsgiComposeParams()
        p.is_debug = 1
        for name, v in D.k5_views(W, H):
            src = ctx.upload(v)
            ctx.ssgi_compose(None, src, None, out, params=p)
            assert _same(out.download(), D.oracle.ssgi_compose_debug(v, (W, H))), name
            src.free()
    finally:
        ctx.close()


class _Scene:
    def __init__(self, ctx):
        self.ctx, self.depth, self.gbuffer, self.velocity = ctx, None, None, None

    def load(self, fr):
        for p in (self.depth, self.gbuffer, self.velocity):
            if p is not None:
                p.free()
        self.depth, self.gbuffer, self.velocity = self.ctx.upload(fr["depth"]), self.ctx.upload(fr["gbuffer"]), self.ctx.upload(fr["velocity"])


class _Composer:
    def __init__(self, ctx, w, h):
        self.ctx, self.width, self.height = ctx, w, h
        self.inputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)
        self.outputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)


class _Cam:
    u = None

    def uniforms(self):
        return self.u


@pytest.mark.parametrize("cls,opts", [(effects.SSGIEffect, {}), (effects.SSGIEffect, {"resolutionScale": 0.5}),
                                      (effects.SSGIEffect, {"denoiseMode": "temporal"}), (effects.SSREffect, {})],
                         ids=["ssgi", "ssgi-scale0.5", "ssgi-temporal", "ssr"])
def test_effect_views_switch_between_frames(built, cls, opts):
    """views switched frame by frame (chain planes, scene planes, G-buffer channels, an unknown string, back to the denoiser's texture):
    K5 equals the oracle's debug branch on the shown plane, isDebug follows the reference's rule, and the chain's planes stay byte-identical
    to an effect that never selected a view (selecting a view resets nothing)"""
    W, H = 160, 96
    inp = ch.make_inputs(W, H, 8)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        scene, cam = _Scene(ctx), _Cam()
        cam.u = inp.frames[0]["cam"]
        comp, comp0 = _Composer(ctx, W, H), _Composer(ctx, W, H)
        fx, fx0 = cls(comp, scene, cam, dict(opts)), cls(comp0, scene, cam, dict(opts))
        den = fx.outputTexture
        views = [lambda: fx._chain.output(1), lambda: scene.depth, lambda: "normal", lambda: "bogus", lambda: fx._chain.output(4),
                 lambda: scene.velocity, lambda: scene.gbuffer, lambda: den]
        for t, fr in enumerate(inp.frames):
            scene.load(fr)  # the host's planes of this frame (a view holds the plane itself)
            fx.outputTexture = views[t]()
            fx.outputTexture = None  # falsy: ignored
            assert fx.isDebug == (t != len(views) - 1)
            comp.inputBuffer.upload(fr["direct"])
            comp0.inputBuffer.upload(fr["direct"])
            cam.u = fr["cam"]
            fx.update(None, comp.inputBuffer)
            fx0.update(None, comp0.inputBuffer)
            got = comp.outputBuffer.download()
            if isinstance(views[t](), str):
                mode = abi.GBUFFER_DEBUG_MODES.index(views[t]()) if views[t]() in abi.GBUFFER_DEBUG_MODES else -1
                shown = D.oracle.gbuffer_debug(mode, fr["gbuffer"])
                assert fx.outputTexture is fx.gBufferDebugTarget and fx.gBufferDebugTarget.download().tobytes() == shown.tobytes()
            else:
                p = fx.outputTexture
                shown = (p.download() if hasattr(p, "download") else _download(ctx, p))
            if fx.isDebug:
                assert _same(got, D.oracle.ssgi_compose_debug(shown, (W, H))), t
            else:
                assert got.tobytes() == comp0.outputBuffer.download().tobytes(), t
                assert fx.gBufferDebugTarget is None
            for which in range(6):
                assert fx._chain.download(which).tobytes() == fx0._chain.download(which).tobytes(), (t, which)
        fx.dispose()
        fx0.dispose()
    finally:
        ctx.close()


def _download(ctx, p: abi.Plane) -> np.ndarray:
    dt, n = engine._NP_OF[p.format]
    out = np.empty((p.height, p.width) if n == 1 else (p.height, p.width, n), dt)
    ctx.sync()
    ctx._chk(ctx.lib.rfx_plane_download(ctx.h, None, C.byref(p), out.ctypes.data_as(C.c_void_p), 0))
    ctx.sync()
    return out


def _traa_params(opts, cam_u, prev_u, keep, moved):
    p = ch.traa_temporal_params(abi.make_camera(cam_u), cam_u["position"], prev_u, keep)
    p.max_blend, p.neighborhood_clamp_intensity, p.confidence_power, p.log_transform = opts.max_blend, opts.neighborhood_clamp_intensity, opts.confidence_power, opts.log_transform
    p.full_accumulate = int(bool(opts.full_accumulate) and not moved)
    return p


VIEWS = [abi.DEBUG_VIEW_OUTPUT + 1, abi.DEBUG_VIEW_OUTPUT + 2, abi.DEBUG_VIEW_OUTPUT + 5, abi.DEBUG_VIEW_DEPTH, abi.DEBUG_VIEW_VELOCITY,
         abi.DEBUG_VIEW_GBUFFER, abi.DEBUG_VIEW_GBUFFER_CHANNEL + 0, abi.DEBUG_VIEW_GBUFFER_CHANNEL + 5]


@pytest.mark.parametrize("fast_math", [True, False], ids=["fast", "per-pass"])
def test_chain_tail_with_a_view_equals_the_passes_by_hand(built, fast_math):
    """each frame a different view: outputs 6 / 7 == ssgi_compose (debug, the view) -> temporal_reproject -> traa_compose by hand; then the
    view is cleared and the chain's outputs equal those of a chain that never had one"""
    W, H = 192, 112
    o = ch.Opts()
    inp = ch.make_inputs(W, H, len(VIEWS) + 2)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast_math)
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, o)
        chain, plain = engine.SsgiChain(ctx, copt), engine.SsgiChain(ctx, copt)
        topt = abi.make_traa_tail_options()
        chain.enable_traa(topt)
        plain.enable_traa(topt)
        k5, out = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
        acc = [ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)]
        dbg = ctx.alloc(abi.FMT_RGBA32F, W, H)
        pd = abi.SsgiComposeParams()
        pd.is_debug = 1
        keep, prev = 0.0, None
        for t, fr in enumerate(inp.frames):
            view = VIEWS[t] if t < len(VIEWS) else abi.DEBUG_VIEW_NONE
            chain.set_debug_view(view)
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            cam = abi.make_camera(fr["cam"])
            chain.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            plain.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            if view == abi.DEBUG_VIEW_NONE:  # the TRAA history differs (it accumulated the debug images); the chain's own planes do not
                for which in range(6):
                    assert chain.download(which).tobytes() == plain.download(which).tobytes(), (t, which)
            else:
                if view >= abi.DEBUG_VIEW_GBUFFER_CHANNEL:
                    ctx.gbuffer_debug(view - abi.DEBUG_VIEW_GBUFFER_CHANNEL, planes[1], dbg)
                    src = dbg
                elif view >= abi.DEBUG_VIEW_DEPTH:
                    src = {abi.DEBUG_VIEW_DEPTH: planes[0], abi.DEBUG_VIEW_VELOCITY: planes[2], abi.DEBUG_VIEW_GBUFFER: planes[1]}[view]
                else:
                    src = chain.output(view)
                ctx.ssgi_compose(planes[0], src, planes[3], k5, params=pd)
                tp = _traa_params(topt, fr["cam"], prev or fr["cam"], keep, fr["moved"])
                ctx.temporal_reproject(tp, k5, planes[2], acc[(t + 1) & 1], None, acc[t & 1], None)
                ctx.traa_compose(acc[t & 1], out)
                assert chain.download(7).tobytes() == acc[t & 1].download().tobytes(), (t, view)
                assert chain.download(6).tobytes() == out.download().tobytes(), (t, view)
                for which in range(6):  # the view changes nothing before the tail
                    assert chain.download(which).tobytes() == plain.download(which).tobytes(), (t, which)
            keep, prev = 1.0, fr["cam"]
            for p in planes:
                p.free()
        chain.close()
        plain.close()
    finally:
        ctx.close()


def test_chain_debug_view_cleared_restores_bytes(built):
    """a view selected for two frames and then cleared: from the frame after, outputs 0..5 equal a chain that never had one, and K9 equals
    that chain's once the TRAA history has been replaced (a reset of both)"""
    W, H = 160, 96
    inp = ch.make_inputs(W, H, 4)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, ch.Opts())
        a, b = engine.SsgiChain(ctx, copt), engine.SsgiChain(ctx, copt)
        for c in (a, b):
            c.enable_traa()
        for t, fr in enumerate(inp.frames):
            a.set_debug_view(abi.DEBUG_VIEW_GBUFFER_CHANNEL + 2 if t < 2 else abi.DEBUG_VIEW_NONE)
            if t == 2:
                a.reset()
                b.reset()
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            for c in (a, b):
                c.render(abi.make_camera(fr["cam"]), *planes, fr["cam"]["position"], fr["moved"])
            if t >= 2:
                for which in range(8):
                    assert a.download(which).tobytes() == b.download(which).tobytes(), (t, which)
            for p in planes:
                p.free()
        a.close()
        b.close()
    finally:
        ctx.close()


def test_chain_debug_view_arguments(built):
    inp = ch.make_inputs(64, 64, 1)
    ctx = engine.Context(0, inp.blue)
    try:
        chain = engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts()))
        for bad in (-2, 6, 7, 11, 15, 22):
            with pytest.raises(abi.RfxError):
                chain.set_debug_view(bad)
        for good in (abi.DEBUG_VIEW_NONE, 0, 1, 5, 8, 10, 16, 21):
            chain.set_debug_view(good)
        chain.close()
    finally:
        ctx.close()


def _inprocess(ctx, chains):
    lib, n = ctx.lib, len(chains)
    groups = []
    for r in range(n):
        g = C.c_void_p()
        ctx._chk(lib.rfx_group_create_inprocess(ctx.h, r, n, C.byref(g)))
        groups.append(g)
    ga = (C.c_void_p * n)(*[g.value for g in groups])
    ca = (C.c_void_p * n)(*[c.h.value for c in chains])
    return lib.rfx_group_attach_chains_inprocess(ga, ca, n), groups


def test_group_refuses_debug_views(built):
    """a chain with a view cannot join a group of n > 1, and a chain in one cannot take a view; clearing is always accepted"""
    W, H = 128, 160
    inp = ch.make_inputs(W, H, 1)
    ctx = engine.Context(0, inp.blue)
    try:
        copt = ch.chain_options(inp, ch.Opts())
        chains = [engine.SsgiChain(ctx, copt) for _ in range(2)]
        chains[1].set_debug_view(abi.DEBUG_VIEW_DEPTH)
        st, groups = _inprocess(ctx, chains)
        assert st == abi.ERR_UNSUPPORTED
        for g in groups:
            ctx.lib.rfx_group_destroy(g)
        chains[1].set_debug_view(abi.DEBUG_VIEW_NONE)
        st, groups = _inprocess(ctx, chains)
        assert st == abi.RFX_OK
        assert ctx.lib.rfx_ssgi_chain_set_debug_view(chains[0].h, abi.DEBUG_VIEW_GBUFFER_CHANNEL) == abi.ERR_UNSUPPORTED
        assert ctx.lib.rfx_ssgi_chain_set_debug_view(chains[0].h, abi.DEBUG_VIEW_NONE) == abi.RFX_OK
        for g in groups:
            ctx.lib.rfx_group_destroy(g)
        for c in chains:
            c.close()
    finally:
        ctx.close()


def test_denoiser_texture_set_back_after_a_resize_ends_debug_mode(built):
    """the denoiser's texture is one object for the effect's life (as denoiser.texture in the reference): held across a resolutionScale
    change and set back, it ends debug mode and K5 composes the new chain's plane; a plane that has been freed is refused"""
    W, H = 128, 80
    inp = ch.make_inputs(W, H, 2)
    ctx = engine.Context(0, inp.blue)
    try:
        scene, cam = _Scene(ctx), _Cam()
        cam.u = inp.frames[0]["cam"]
        comp, comp0 = _Composer(ctx, W, H), _Composer(ctx, W, H)
        fx = effects.SSGIEffect(comp, scene, cam)
        den, dnb = fx.outputTexture, fx.chainTexture(4)
        fx.outputTexture = "metalness"
        old_target = fx.gBufferDebugTarget
        fx.resolutionScale = 0.5  # a new chain and a new debug target
        fx0 = effects.SSGIEffect(comp0, scene, cam, {"resolutionScale": 0.5})
        with pytest.raises(abi.RfxError):
            fx.outputTexture = old_target
        fx.outputTexture = dnb
        assert fx.isDebug and fx.gBufferDebugTarget is None and fx.outputTexture is dnb
        fx.outputTexture = den
        assert not fx.isDebug and fx.outputTexture is den
        for fr in inp.frames:
            scene.load(fr)
            cam.u = fr["cam"]
            for c, e in ((comp, fx), (comp0, fx0)):
                c.inputBuffer.upload(fr["direct"])
                e.update(None, c.inputBuffer)
            assert comp.outputBuffer.download().tobytes() == comp0.outputBuffer.download().tobytes()
            assert _download(ctx, fx.outputTexture).tobytes() == fx0._chain.download(0).tobytes()
        fx.dispose()
        fx0.dispose()
    finally:
        ctx.close()
