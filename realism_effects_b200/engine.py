"""Thin Python host layer over the C ABI (include/rfx.h): context, device planes, pass launches.

This is plumbing, not the product: every method forwards to one `rfx_*` entry point of
csrc/librfx.so and raises RfxError on a non-zero status (like the JS wrapper of INTEGRATION.md
would throw).  There is no CPU path here.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi
from .abi import (FMT_R32F, FMT_RGBA8, FMT_RGBA16F, FMT_RGBA32F, Plane, RfxError)


def _fmt_of(a: np.ndarray) -> int:
    if a.ndim == 2 and a.dtype == np.float32:
        return FMT_R32F
    if a.ndim == 3 and a.shape[2] == 4:
        if a.dtype == np.float32:
            return FMT_RGBA32F
        if a.dtype in (np.float16, np.uint16):
            return FMT_RGBA16F
        if a.dtype == np.uint8:
            return FMT_RGBA8
    raise RfxError(f"no plane format for array {a.shape} {a.dtype}")


_NP_OF = {FMT_R32F: (np.float32, 1), FMT_RGBA32F: (np.float32, 4), FMT_RGBA16F: (np.float16, 4), FMT_RGBA8: (np.uint8, 4)}


class DevPlane:
    """An rfx_plane owned by a Context."""

    def __init__(self, ctx: "Context", fmt: int, width: int, height: int):
        self.ctx = ctx
        self.p = Plane()
        ctx._chk(ctx.lib.rfx_plane_alloc(ctx.h, fmt, width, height, C.byref(self.p)))
        self.owned = True

    @property
    def width(self):
        return self.p.width

    @property
    def height(self):
        return self.p.height

    @property
    def format(self):
        return self.p.format

    def ref(self):
        return C.byref(self.p)

    def upload(self, a: np.ndarray, stream=None):
        a = np.ascontiguousarray(a)
        assert _fmt_of(a) == self.p.format and a.shape[0] == self.p.height and a.shape[1] == self.p.width, (a.shape, a.dtype)
        self.ctx._chk(self.ctx.lib.rfx_plane_upload(self.ctx.h, stream, self.ref(), a.ctypes.data_as(C.c_void_p), 0))
        self.ctx.sync()
        return self

    def download(self) -> np.ndarray:
        dt, ch = _NP_OF[self.p.format]
        shape = (self.p.height, self.p.width) if ch == 1 else (self.p.height, self.p.width, ch)
        out = np.empty(shape, dt)
        self.ctx.sync()
        self.ctx._chk(self.ctx.lib.rfx_plane_download(self.ctx.h, None, self.ref(), out.ctypes.data_as(C.c_void_p), 0))
        self.ctx.sync()
        return out

    def clear(self):
        self.ctx._chk(self.ctx.lib.rfx_plane_clear(self.ctx.h, None, self.ref()))

    def free(self):
        if self.owned and self.p.ptr:
            self.ctx.lib.rfx_plane_free(self.ctx.h, self.ref())
            self.owned = False


def _r(p):
    return None if p is None else (p.ref() if isinstance(p, DevPlane) else C.byref(p))


class Context:
    def __init__(self, device: int = 0, blue_noise: np.ndarray | None = None):
        self.lib = abi.lib()
        h = C.c_void_p()
        st = self.lib.rfx_ctx_create(device, C.byref(h))
        if st != 0:
            raise RfxError(f"rfx_ctx_create(device={device}) failed with status {st} (is a CUDA device visible?)")
        self.h = h
        self.device = device
        self._keep = []
        if blue_noise is None:
            from .synth import load_blue_noise

            blue_noise = load_blue_noise()
        self.set_blue_noise(blue_noise)

    def _chk(self, st: int):
        if st != 0:
            raise RfxError(f"rfx status {st}: {self.lib.rfx_last_error(self.h).decode()}")

    def close(self):
        if self.h:
            self.lib.rfx_ctx_destroy(self.h)
            self.h = None

    def sync(self):
        self._chk(self.lib.rfx_ctx_sync(self.h))

    @property
    def stream(self):
        return self.lib.rfx_ctx_stream(self.h)

    @property
    def launch_count(self) -> int:
        return int(self.lib.rfx_launch_count(self.h))

    def set_fast_math(self, enable: bool):
        """True (default): SFU-pipe kernel variants; False: exact-libm variants (bit-level parity with the oracle)."""
        self._chk(self.lib.rfx_ctx_set_fast_math(self.h, int(enable)))

    def set_blue_noise(self, rgba8: np.ndarray):
        a = np.ascontiguousarray(rgba8, dtype=np.uint8)
        self._chk(self.lib.rfx_blue_noise_set(self.h, a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0]))

    def set_env(self, map_f16: np.ndarray, marginal: np.ndarray | None, conditional: np.ndarray | None, total_sum: float):
        m = np.ascontiguousarray(map_f16)
        assert m.dtype in (np.float16, np.uint16) and m.ndim == 3 and m.shape[2] == 4
        d = abi.EnvDesc()
        d.map_rgba16f = m.ctypes.data
        d.width, d.height = m.shape[1], m.shape[0]
        keep = [m]
        if marginal is not None:
            mg = np.ascontiguousarray(marginal, np.float32)
            cd = np.ascontiguousarray(conditional, np.float32)
            d.marginal, d.conditional = mg.ctypes.data, cd.ctypes.data
            keep += [mg, cd]
        whole = float(int(total_sum))  # ~~totalSumValue (EquirectHdrInfoUniform.js:346-349)
        d.total_sum_whole = float(np.float32(whole))
        d.total_sum_decimal = float(np.float32(total_sum - whole))
        self._chk(self.lib.rfx_env_set(self.h, C.byref(d)))
        self._env_shape = (m.shape[0], m.shape[1])

    def build_env(self, map_f16: np.ndarray, flip_y: bool = False):
        """env map + importance-sampling tables built on the device (rfx_env_build)"""
        m = np.ascontiguousarray(map_f16)
        assert m.dtype in (np.float16, np.uint16) and m.ndim == 3 and m.shape[2] == 4
        self._chk(self.lib.rfx_env_build(self.h, m.ctypes.data, m.shape[1], m.shape[0], int(flip_y)))
        self._env_shape = (m.shape[0], m.shape[1])

    def env_tables(self):
        """(marginal[H], conditional[H, W], totalSum) of the current environment, downloaded"""
        h, w = self._env_shape
        marg, cond, tot = np.empty(h, np.float32), np.empty((h, w), np.float32), C.c_double()
        self._chk(self.lib.rfx_env_tables_download(self.h, marg.ctypes.data, cond.ctypes.data, C.byref(tot)))
        return marg, cond, float(tot.value)

    def clear_env(self):
        self._chk(self.lib.rfx_env_clear(self.h))

    def alloc(self, fmt: int, width: int, height: int) -> DevPlane:
        return DevPlane(self, fmt, width, height)

    def upload(self, a: np.ndarray) -> DevPlane:
        a = np.ascontiguousarray(a)
        return DevPlane(self, _fmt_of(a), a.shape[1], a.shape[0]).upload(a)

    # ---- pass launches (one per reference fullscreen draw) -----------------------------------
    def ssgi_trace(self, p, depth, gbuffer, velocity, direct_light, accumulated, out, rows=(0, 0), stream=None):
        self._chk(self.lib.rfx_ssgi_trace_launch(self.h, stream, C.byref(p), _r(depth), _r(gbuffer), _r(velocity), _r(direct_light),
                                                 _r(accumulated), _r(out), rows[0], rows[1]))

    def temporal_reproject(self, p, inp, velocity, hist0, hist1, out0, out1, rows=(0, 0), stream=None):
        self._chk(self.lib.rfx_temporal_reproject_launch(self.h, stream, C.byref(p), _r(inp), _r(velocity), _r(hist0), _r(hist1), _r(out0),
                                                         _r(out1), rows[0], rows[1]))

    def poisson_denoise(self, p, depth, gbuffer_or_normal, in0, in1, out0, out1, rows=(0, 0), stream=None):
        self._chk(self.lib.rfx_poisson_denoise_launch(self.h, stream, C.byref(p), _r(depth), _r(gbuffer_or_normal), _r(in0), _r(in1), _r(out0),
                                                      _r(out1), rows[0], rows[1]))

    def gi_compose(self, p, depth, gbuffer, diffuse_gi, specular_gi, out, rows=(0, 0), stream=None, scene=None):
        self._chk(self.lib.rfx_gi_compose_launch(self.h, stream, C.byref(p), _r(depth), _r(gbuffer), _r(diffuse_gi), _r(specular_gi), _r(scene), _r(out),
                                                 rows[0], rows[1]))

    def ssgi_compose(self, depth, gi, scene, out, rows=(0, 0), stream=None, params=None):
        """params: abi.SsgiComposeParams (scene fog / isDebug) or None.  With params.is_debug, gi is the debug view: any R32F, RGBA16F or
        RGBA32F plane of any size (depth / scene are not read and may be None)"""
        self._chk(self.lib.rfx_ssgi_compose_launch(self.h, stream, C.byref(params) if params is not None else None, _r(depth), _r(gi), _r(scene), _r(out),
                                                   rows[0], rows[1]))

    def hbao(self, p, depth, out, rows=(0, 0), stream=None, normal=None):
        """out may be smaller than depth (AO resolutionScale; p.resolution = its unrounded size, {0, 0} = out's size);
        normal: RGBA8 view-space normal plane (NormalPass layout, p.view_matrix turns it to world space) or None"""
        self._chk(self.lib.rfx_hbao_launch_ex(self.h, stream, C.byref(p), _r(depth), _r(normal), _r(out), rows[0], rows[1]))

    def hbao_horizon(self, p, depth, out, normal=None, stream=None):
        """K6h, horizon-march AO (abi.HbaoHorizonParams): K6's planes and output layout; normal: RGBA8 view-space normal plane of depth's
        size or None"""
        self._chk(self.lib.rfx_hbao_horizon_launch(self.h, stream, C.byref(p), _r(depth), _r(out), _r(normal)))

    def ao_compose(self, p, depth, ao, inp, out, rows=(0, 0), stream=None):
        self._chk(self.lib.rfx_ao_compose_launch(self.h, stream, C.byref(p), _r(depth), _r(ao), _r(inp), _r(out), rows[0], rows[1]))

    def motion_blur(self, p, velocity, inp, out, rows=(0, 0), stream=None):
        self._chk(self.lib.rfx_motion_blur_launch(self.h, stream, C.byref(p), _r(velocity), _r(inp), _r(out), rows[0], rows[1]))

    def gbuffer_debug(self, mode, gbuffer, out, rows=(0, 0), stream=None):
        """GBufferDebugPass: channel `mode` (abi.GBUFFER_DEBUG_MODES index; any other value shows emissive) of the packed G-buffer, RGBA32F"""
        self._chk(self.lib.rfx_gbuffer_debug_launch(self.h, stream, int(mode), _r(gbuffer), _r(out), rows[0], rows[1]))

    def traa_compose(self, acc, out, rows=(0, 0), stream=None):
        self._chk(self.lib.rfx_traa_compose_launch(self.h, stream, _r(acc), _r(out), rows[0], rows[1]))

    def effects(self, p, inp, depth, velocity, out, rows=(0, 0), stream=None):
        """merged cosmetic effects (abi.make_effects_params): Sharpness / LensDistortion / GradualBackground / Sparkle in one launch"""
        self._chk(self.lib.rfx_effects_launch(self.h, stream, C.byref(p), _r(inp), _r(depth), _r(velocity), _r(out), rows[0], rows[1]))

    def taa(self, p, inp, history, out, rows=(0, 0), stream=None):
        self._chk(self.lib.rfx_taa_launch(self.h, stream, C.byref(p), _r(inp), _r(history), _r(out), rows[0], rows[1]))

    def gbuffer_ingest(self, albedo, normal, material, emissive, motion, depth, out_gbuffer, out_velocity, *, motion_scale=(1.0, 1.0),
                       normalize_normals=True, rows=(0, 0), stream=None):
        """conventional SoA planes -> the reference's packed gBuffer / velocity planes (rfx_gbuffer_ingest_launch)"""
        p = abi.IngestParams()
        p.motion_scale[:] = [float(motion_scale[0]), float(motion_scale[1])]
        p.normalize_normals = int(bool(normalize_normals))
        self._chk(self.lib.rfx_gbuffer_ingest_launch(self.h, stream, C.byref(p), _r(albedo), _r(normal), _r(material), _r(emissive), _r(motion),
                                                     _r(depth), _r(out_gbuffer), _r(out_velocity), rows[0], rows[1]))


class SsgiChain:
    """Native SSGI chain (rfx_ssgi_chain): K1 -> K2 -> K3 x 2*iterations -> K4 with history."""

    def __init__(self, ctx: Context, opt: abi.ChainOptions):
        self.ctx = ctx
        self.opt = opt
        self.traa = None
        h = C.c_void_p()
        ctx._chk(ctx.lib.rfx_ssgi_chain_create(ctx.h, C.byref(opt), C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            self.ctx.lib.rfx_ssgi_chain_destroy(self.h)
            self.h = None

    def reset(self):
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_reset(self.h))

    def set_options(self, opt: abi.ChainOptions):
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_set_options(self.h, C.byref(opt)))
        self.opt = opt

    def enable_traa(self, options: "abi.TraaTailOptions | None" = None, enable: bool = True):
        """TRAA frame tail (K5 -> TRAA -> K9 after K4, include/rfx.h: rfx_ssgi_chain_enable_traa): outputs 6 (the K9 frame) and 7 (the
        TRAA accumulated plane).  options: abi.make_traa_tail_options(...) (default: TRAAEffect's values, no fog); enable=False turns it off.
        Enabling again replaces the options and resets the TRAA history."""
        if not enable:
            self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_enable_traa(self.h, None))
            self.traa = None
            return
        self.traa = options if options is not None else abi.make_traa_tail_options()
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_enable_traa(self.h, C.byref(self.traa)))

    def set_debug_view(self, view: int):
        """the TRAA tail's K5 shows `view` (abi.DEBUG_VIEW_*; include/rfx.h: rfx_ssgi_chain_set_debug_view) instead of composed"""
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_set_debug_view(self.h, int(view)))

    @staticmethod
    def _frame(cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved) -> abi.SsgiFrame:
        f = abi.SsgiFrame()
        f.cam = cam
        f.depth = C.pointer(depth.p)
        f.gbuffer = C.pointer(gbuffer.p)
        f.velocity = C.pointer(velocity.p)
        f.direct_light = C.pointer(direct_light.p) if direct_light is not None else None
        f.camera_pos[:] = [float(x) for x in camera_pos]
        f.camera_moved = int(camera_moved)
        return f

    def render(self, cam: abi.CameraS, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved: bool, stream=None):
        f = self._frame(cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved)
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_render(self.h, stream, C.byref(f)))

    def output(self, which: int = 0) -> Plane:
        """0 composed, 1 ssgiOut, 2/3 trOut, 4/5 dnB; with the TRAA tail on, 6 the K9 output and 7 the TRAA accumulated plane"""
        p = Plane()
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_output(self.h, which, C.byref(p)))
        return p

    def download(self, which: int = 0) -> np.ndarray:
        p = self.output(which)
        dt, ch = _NP_OF[p.format]
        out = np.empty((p.height, p.width, ch), dt)
        self.ctx.sync()
        self.ctx._chk(self.ctx.lib.rfx_plane_download(self.ctx.h, None, C.byref(p), out.ctypes.data_as(C.c_void_p), 0))
        self.ctx.sync()
        return out

    PROFILE_SLOTS = ("K1_ssgi_trace", "K2_temporal_reproject", "K3_poisson_pass0", "K3_poisson_pass1plus", "K4_gi_compose")

    def set_profiling(self, enable: bool):
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_set_profiling(self.h, int(enable)))

    def get_profile(self) -> dict:
        """{slot: (total_ms, launches)} for the frames rendered since the last call."""
        ms = (C.c_double * 5)()
        n = (C.c_uint64 * 5)()
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_get_profile(self.h, ms, n))
        return {k: (float(ms[i]), int(n[i])) for i, k in enumerate(self.PROFILE_SLOTS)}

    def render_host(self, hf: abi.SsgiHostFrame):
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_render_host(self.h, C.byref(hf)))

    def submit_host(self, hf: abi.SsgiHostFrame):
        """Pipelined host path: enqueue H2D -> chain -> D2H for one frame and return (include/rfx.h: rfx_ssgi_chain_submit_host)."""
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_submit_host(self.h, C.byref(hf)))

    def wait_host(self, max_in_flight: int = 0):
        self.ctx._chk(self.ctx.lib.rfx_ssgi_chain_wait_host(self.h, int(max_in_flight)))


def ao_chain_options(width: int, height: int, options: dict | None = None, horizon: bool = False) -> abi.AoChainOptions:
    """rfx_ao_chain_options from HBAOEffect's option table (effects.defaultAOOptions), or HorizonAOEffect's with horizon=True
    (effects.defaultHorizonAOOptions); missing keys take those defaults.  `blueNoiseStart` is the AO pass's start (the effect's option),
    `denoiseBlueNoiseStart` the denoiser's (PoissonDenoisePass's, 1234567)."""
    from . import effects

    o = {**(effects.defaultHorizonAOOptions if horizon else effects.defaultAOOptions), **(options or {})}
    if horizon:
        effects.check_horizon_ao_options(o)
    c = abi.AoChainOptions()
    c.width, c.height = int(width), int(height)
    c.algorithm = abi.AO_HORIZON if horizon else abi.AO_HBAO
    c.resolution_scale = float(o["resolutionScale"])
    c.use_normal_plane = int(bool(o.get("useNormalPass") or o.get("normalTexture") is not None))
    c.spp, c.distance = int(o.get("spp", 0)), float(o["distance"])
    c.distance_power, c.bias, c.thickness = float(o.get("distancePower", 0.0)), float(o.get("bias", 0.0)), float(o.get("thickness", 0.0))
    c.directions, c.steps = int(o.get("directions", 1)), int(o.get("steps", 1))
    c.angle_bias, c.intensity, c.max_radius_pixels = float(o.get("angleBias", 0.0)), float(o.get("intensity", 1.0)), float(o.get("maxRadiusPixels", 1.0))
    c.iterations, c.radius, c.phi = int(o["iterations"]), float(o["radius"]), float(o["phi"])
    c.luma_phi, c.depth_phi, c.normal_phi = float(o["lumaPhi"]), float(o["depthPhi"]), float(o["normalPhi"])
    c.power = float(o["power"])
    c.color[:] = [float(x) for x in o["color"]]
    c.blue_noise_start = int(o.get("blueNoiseStart", 1234567))
    c.denoise_blue_noise_start = int(o.get("denoiseBlueNoiseStart", 1234567))
    return c


class AoChain:
    """Native AO chain (rfx_ao_chain): K6 or K6h -> K3 x 2*iterations -> K7 in one call, the launches of HBAOEffect.update /
    HorizonAOEffect.update.  Options: ao_chain_options(...)."""

    def __init__(self, ctx: Context, opt: abi.AoChainOptions):
        self.ctx, self.opt = ctx, opt
        h = C.c_void_p()
        ctx._chk(ctx.lib.rfx_ao_chain_create(ctx.h, C.byref(opt), C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            self.ctx.lib.rfx_ao_chain_destroy(self.h)
            self.h = None

    def reset(self):
        self.ctx._chk(self.ctx.lib.rfx_ao_chain_reset(self.h))

    def set_options(self, opt: abi.AoChainOptions):
        self.ctx._chk(self.ctx.lib.rfx_ao_chain_set_options(self.h, C.byref(opt)))
        self.opt = opt

    @staticmethod
    def _frame(cam_u: dict, depth, velocity, normal=None, inp=None, out=None) -> abi.AoFrame:
        """cam_u: camera uniforms (synth.Camera.uniforms()); planes: DevPlane (or objects with `.p`), normal / inp / out may be None"""
        f = abi.AoFrame()
        for k in ("projection", "projection_inverse", "camera_matrix_world", "view_matrix"):
            abi.set_f16(getattr(f, k), cam_u[k])
        ptr = lambda p: None if p is None else C.pointer(p.p)  # noqa: E731
        f.depth, f.velocity, f.normal, f.input, f.output = ptr(depth), ptr(velocity), ptr(normal), ptr(inp), ptr(out)
        return f

    def render(self, cam_u: dict, depth, velocity, normal=None, inp=None, out=None, stream=None):
        """one frame; out=None skips K7"""
        f = self._frame(cam_u, depth, velocity, normal, inp, out)
        self.ctx._chk(self.ctx.lib.rfx_ao_chain_render(self.h, stream, C.byref(f)))

    def output(self, which: int = 1) -> Plane:
        """0 the AO target, 1 the denoised plane K7 composes (the AO target with iterations 0)"""
        p = Plane()
        self.ctx._chk(self.ctx.lib.rfx_ao_chain_output(self.h, which, C.byref(p)))
        return p

    def download(self, which: int = 1) -> np.ndarray:
        p = self.output(which)
        out = np.empty((p.height, p.width, 4), np.float16)
        self.ctx.sync()
        self.ctx._chk(self.ctx.lib.rfx_plane_download(self.ctx.h, None, C.byref(p), out.ctypes.data_as(C.c_void_p), 0))
        self.ctx.sync()
        return out
