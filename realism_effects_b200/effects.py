"""Host-side mirror of the reference's plugin surface (src/index.js:16-31) over the C ABI.

The reference's host language (JavaScript on a WebGL renderer) has no toolchain in this image, so the
host side above the C ABI is written here in Python with the reference's class names, constructor
signatures, option names/defaults and methods; `js/` holds the same classes as ES modules over the
N-API shim for a box that has Node (INTEGRATION.md).  Every compute call below ends in one `rfx_*`
entry point of csrc/librfx.so — there is no CPU path.

What stands in for three.js / postprocessing objects:
  composer  : any object with `.ctx` (engine.Context), `.width/.height`, `.inputBuffer` (DevPlane RGBA16F, the
              scene colour = directLight) and `.outputBuffer` (DevPlane RGBA16F)
  scene     : any object with `.gbuffer`, `.depth` (packed G-buffer + depth planes, the output layout of
              GBufferPass, src/gbuffer/GBufferPass.js:33-44) and `.velocity` (VelocityDepthNormalPass layout)
              — rasterising meshes into those planes is out of scope (SURVEY.md §2, K10/K11)
  camera    : synth.Camera or any object with `.uniforms()` (three.js matrices as float32 column-major)
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from . import abi, engine

# ---------------------------------------------------------------------------------------------------
# option tables (verbatim defaults)
# ---------------------------------------------------------------------------------------------------
defaultSSGIOptions = dict(  # src/ssgi/SSGIOptions.js:26-48
    mode="ssgi", distance=10, thickness=10, denoiseIterations=1, denoiseKernel=2, denoiseDiffuse=10, denoiseSpecular=10, radius=3, phi=0.5,
    lumaPhi=5, depthPhi=2, normalPhi=50, roughnessPhi=50, specularPhi=50, envBlur=0.5, importanceSampling=True, steps=20, refineSteps=5,
    resolutionScale=1, missedRays=False, outputTexture=None)
defaultTemporalReprojectPassOptions = dict(  # src/temporal-reproject/TemporalReprojectPass.js:17-32
    dilation=False, fullAccumulate=False, neighborhoodClamp=False, neighborhoodClampRadius=1, neighborhoodClampIntensity=1, maxBlend=1,
    logTransform=False, depthDistance=2, worldDistance=4, reprojectSpecular=False, renderTarget=None, copyTextures=True, confidencePower=0.75,
    inputType="diffuse")
defaultPoissonBlurOptions = dict(  # src/denoise/pass/PoissonDenoisePass.js:16-24
    iterations=1, radius=3, phi=0.5, lumaPhi=5, depthPhi=2, normalPhi=3.25, inputType="diffuseSpecular")
defaultAOOptions = dict(  # src/ao/AOEffect.js:8-21
    resolutionScale=1, spp=8, distance=2, distancePower=1, power=2, bias=40, thickness=0.075, color=(0.0, 0.0, 0.0), useNormalPass=False,
    velocityDepthNormalPass=None, normalTexture=None, **defaultPoissonBlurOptions)
defaultMotionBlurOptions = dict(intensity=1, jitter=1, samples=16)  # src/motion-blur/MotionBlurEffect.js:14

_HIGHEST_SIGNED_INT = 0x7FFFFFFF


class BlueNoiseIndex:
    """The `blueNoiseIndex` uniform of setupBlueNoise (src/utils/BlueNoiseUtils.js:17-33): advances on every read.
    `start` pins the reference's Math.random() seed."""

    def __init__(self, start: int = 1234567):
        self.start, self.i = int(start), 0

    @property
    def value(self) -> int:
        self.i = (self.start + self.i + 1) % _HIGHEST_SIGNED_INT
        return self.i


def _did_camera_move(cam_u: dict, last: dict | None) -> bool:
    """src/utils/SceneUtils.js:17-27 (position / orientation compared with small epsilons)"""
    if last is None:
        return True
    a, b = np.asarray(cam_u["camera_matrix_world"], np.float64), np.asarray(last["camera_matrix_world"], np.float64)
    return bool(np.abs(a[12:15] - b[12:15]).max() > 1e-6 or np.abs(a[:12] - b[:12]).max() > 1e-6)


class _Reactive:
    """Every option key becomes a get/set property of the effect (makeOptionsReactive)."""

    _options: dict

    def __getattr__(self, k):
        o = self.__dict__.get("_options")
        if o is not None and k in o:
            return o[k]
        raise AttributeError(k)

    def __setattr__(self, k, v):
        o = self.__dict__.get("_options")
        if o is not None and k in o and not k.startswith("_"):
            if o[k] != v:
                o[k] = v
                self._option_changed(k)
            return
        object.__setattr__(self, k, v)

    def _option_changed(self, k):  # pragma: no cover - overridden
        pass


# ---------------------------------------------------------------------------------------------------
def _debug_state(value):
    """What SSGIEffect's outputTexture setter does with `value` (src/ssgi/SSGIEffect.js:228-251): None for a falsy value (the setter returns
    early), ("gbuffer", mode) for a string (GBufferDebugPass mode = its index in the mode list, -1 when unknown, which shows emissive),
    ("texture", None) for a plane"""
    if value is None or (isinstance(value, str) and not value):
        return None
    if isinstance(value, str):
        return ("gbuffer", abi.GBUFFER_DEBUG_MODES.index(value) if value in abi.GBUFFER_DEBUG_MODES else -1)
    return ("texture", None)


def _plane_ptr(p) -> int:
    return int((p.p if hasattr(p, "p") else p).ptr or 0)


class _ChainTexture(abi.Plane):
    """Chain output `which` of one effect as an object that outlives the chain: the effect refreshes its fields from the current chain
    whenever it hands it out, so a host can hold it across setSize / resolutionScale changes and set it back (the reference's
    denoiser.texture is one object for the effect's life)."""

    def __init__(self, owner, which: int):
        super().__init__()
        self.owner, self.which = owner, which


# ---------------------------------------------------------------------------------------------------
class VelocityDepthNormalPass:
    """src/temporal-reproject/pass/VelocityDepthNormalPass.js:66-194.  The reference rasterises the scene into
    (uv motion, packed oct normal, depth); here the plane is supplied by the host (`scene.velocity`)."""

    needsSwap = False

    def __init__(self, scene, camera):
        self._scene, self._camera = scene, camera
        self.lastVelocityTexture = None

    @property
    def texture(self):
        return self._scene.velocity

    @property
    def renderTarget(self):
        return self

    @property
    def depthTexture(self):
        return self._scene.depth

    def setSize(self, width, height):
        pass

    def render(self, renderer=None):
        self.lastVelocityTexture = self._scene.velocity

    def dispose(self):
        pass


class VelocityPass(VelocityDepthNormalPass):
    """src/temporal-reproject/pass/VelocityPass.js:3-7: the same pass object (the host supplies the plane either way)"""


# ---------------------------------------------------------------------------------------------------
class SSGIEffect(_Reactive):
    """new SSGIEffect(composer, scene, camera, options)   (src/ssgi/SSGIEffect.js:27-141; signature per D6)

    update() runs K1 -> K2 -> K3 x 2*denoiseIterations -> K4 natively (rfx_ssgi_chain) and then K5 into
    composer.outputBuffer.  `outputTexture` is the composed GI plane (RGBA32F), the denoiser's texture.

    Debug views (SSGIEffect.js:228-251): setting `outputTexture` to another plane the host holds (a chain output, scene.depth, scene.velocity,
    scene.gbuffer) makes K5 show that plane (isDebug); setting it to one of abi.GBUFFER_DEBUG_MODES (an unknown string shows emissive) renders
    that G-buffer channel with GBufferDebugPass after the chain every frame and shows its target, which the getter then returns.  Setting the
    denoiser's texture back ends debug mode; a falsy value is ignored.  No view resets the temporal history."""

    DefaultOptions = defaultSSGIOptions

    def __init__(self, composer, scene, camera, options=None):
        opts = {**defaultSSGIOptions, **(options or {})}
        if opts["mode"] == "ssr":  # src/ssgi/SSGIEffect.js:70-77
            opts.update(reprojectSpecular=True, neighborhoodClamp=True, inputType="specular")
        else:
            opts.update(reprojectSpecular=[False, True], neighborhoodClamp=[False, True])
        opts.setdefault("denoiseMode", "full")  # Denoiser.js:6-11 (spread into the Denoiser through ...options, SSGIEffect.js:104-108)
        preset = opts.get("preset")
        if isinstance(preset, str):  # src/ssgi/SSGIEffect.js:79-99 (the third case is a second, unreachable "medium" in the reference)
            if preset == "low":
                opts.update(steps=10, refineSteps=2, denoiseMode="full_temporal")
            elif preset == "medium":
                opts.update(steps=20, refineSteps=4, denoiseMode="full")
        if opts["denoiseMode"] not in abi.DENOISE_MODES:
            raise abi.RfxError(f"denoiseMode {opts['denoiseMode']!r}: 'denoised' binds an array of textures to a sampler in the reference and cannot run there; "
                               f"supported: {sorted(abi.DENOISE_MODES)}")
        self.composer, self._scene, self._camera = composer, scene, camera
        self.ctx: engine.Context = composer.ctx
        self.velocityDepthNormalPass = opts.get("velocityDepthNormalPass") or VelocityDepthNormalPass(scene, camera)
        self.isUsingRenderPass = True  # directLight comes from the composer input buffer (useDirectLight)
        self._blue_start = int(opts.pop("blueNoiseStart", 1234567))
        self._last_cam = None
        self._chain = None
        self._chain_textures = [_ChainTexture(self, n) for n in range(6)]  # chainTexture(n); 0 is the denoiser's texture
        self._view = None  # debug view: None (the denoiser's texture), ("output", n), ("plane", plane) or ("gbuffer", mode)
        self.gBufferDebugTarget = None
        self.isDebug = False
        self._options = opts
        self.setSize(composer.width, composer.height)

    # -- native chain ------------------------------------------------------------------------------
    def _chain_options(self) -> abi.ChainOptions:
        o, c = self._options, abi.ChainOptions()
        c.width, c.height = self._size
        c.denoise_iterations, c.steps, c.refine_steps = int(o["denoiseIterations"]), int(o["steps"]), int(o["refineSteps"])
        c.distance, c.thickness, c.env_blur = o["distance"], o["thickness"], o["envBlur"]
        c.radius, c.phi, c.luma_phi, c.depth_phi = o["radius"], o["phi"], o["lumaPhi"], o["depthPhi"]
        c.normal_phi, c.roughness_phi, c.specular_phi = o["normalPhi"], o["roughnessPhi"], o["specularPhi"]
        flags = 0
        if getattr(self.ctx, "has_env", False):
            flags |= abi.SSGI_USE_ENVMAP | (abi.SSGI_IMPORTANCE_SAMPLING if o["importanceSampling"] else 0)
        if o["missedRays"]:
            flags |= abi.SSGI_MISSED_RAYS
        if self.isUsingRenderPass:
            flags |= abi.SSGI_USE_DIRECT_LIGHT
        c.ssgi_flags = flags
        c.mode = abi.MODE_SSR if o["mode"] == "ssr" else abi.MODE_SSGI
        c.blue_noise_start = self._blue_start
        c.denoise_mode = abi.DENOISE_MODES[o["denoiseMode"]]
        c.resolution_scale = float(o["resolutionScale"])
        return c

    def setSize(self, width, height, force=False):
        if not force and getattr(self, "_size", None) == (width, height):
            return
        self._size = (int(width), int(height))
        if self._chain is not None:
            self._chain.close()
        self._chain = engine.SsgiChain(self.ctx, self._chain_options())
        if self.gBufferDebugTarget is not None:  # GBufferDebugPass.setSize at the effect's size
            self.gBufferDebugTarget.free()
            self.gBufferDebugTarget = self.ctx.alloc(abi.FMT_RGBA32F, *self._size)

    def __setattr__(self, k, v):
        if k == "outputTexture":  # SSGIEffect.js:228-251: no reset(), unlike the other setters
            self._set_output_texture(v)
        else:
            super().__setattr__(k, v)

    def _set_output_texture(self, v):
        st = _debug_state(v)
        if st is None:
            return
        kind, mode = st
        if kind == "gbuffer":
            if self.gBufferDebugTarget is None:
                self.gBufferDebugTarget = self.ctx.alloc(abi.FMT_RGBA32F, *self._size)
            self._view = ("gbuffer", mode)
        elif v is not self.gBufferDebugTarget:
            if isinstance(v, _ChainTexture) and v.owner is self:
                n = v.which
            else:
                ptr = _plane_ptr(v)
                if ptr == 0 or (isinstance(v, engine.DevPlane) and not v.owned):
                    raise abi.RfxError("SSGIEffect.outputTexture: the plane has been freed")
                # a chain plane is looked up again every frame: the fast chain re-splits trOut / dnB when they are read
                n = next((i for i in range(6) if _plane_ptr(self._chain.output(i)) == ptr), None)
            if self.gBufferDebugTarget is not None:
                self.gBufferDebugTarget.free()
                self.gBufferDebugTarget = None
            self._view = None if n == 0 else ("output", n) if n is not None else ("plane", v)
        self.isDebug = self._view is not None

    def chainTexture(self, which: int) -> abi.Plane:
        """chain output `which` (0 the denoiser's texture, 1 ssgiOut, 2/3 trOut, 4/5 dnB) as a texture that stays valid across setSize"""
        t, p = self._chain_textures[which], self._chain.output(which)
        C.memmove(C.addressof(t), C.addressof(p), C.sizeof(abi.Plane))
        return t

    def _view_plane(self):
        if self._view is None:
            return self.chainTexture(0)
        kind, x = self._view
        return self.gBufferDebugTarget if kind == "gbuffer" else self.chainTexture(x) if kind == "output" else x

    def _option_changed(self, k):
        if k == "resolutionScale":
            self.setSize(*self._size, force=True)
        elif self._chain is not None:
            self._chain.set_options(self._chain_options())  # setters end with reset() in the reference

    def setEnvironment(self, map_f16, marginal=None, conditional=None, total_sum=1.0):
        """keepEnvMapUpdated (src/ssgi/SSGIEffect.js:309-366): equirect RGBA16F map + CDF tables"""
        self.ctx.set_env(map_f16, marginal, conditional, total_sum)
        self.ctx.has_env = True
        self._chain.set_options(self._chain_options())

    def reset(self):
        self._chain.reset()

    def initialize(self, renderer=None, *args):
        pass

    @property
    def depthTexture(self):
        return self._scene.depth

    @property
    def outputTexture(self):
        return self._view_plane()

    def update(self, renderer=None, inputBuffer=None, deltaTime=None):
        cam_u = self._camera.uniforms()
        moved = _did_camera_move(cam_u, self._last_cam)
        self._last_cam = cam_u
        self.velocityDepthNormalPass.render(renderer)
        scene_buf = inputBuffer if inputBuffer is not None else self.composer.inputBuffer
        self._chain.render(abi.make_camera(cam_u), self._scene.depth, self._scene.gbuffer, self.velocityDepthNormalPass.texture,
                           scene_buf if self.isUsingRenderPass else None, cam_u["position"], moved)
        if self._view is not None and self._view[0] == "gbuffer":  # GBufferDebugPass renders after SSGIPass (SSGIEffect.js:398-399)
            self.ctx.gbuffer_debug(self._view[1], self._scene.gbuffer, self.gBufferDebugTarget)
        if getattr(self.composer, "outputBuffer", None) is not None:  # both modes: SSR composes with inputType "specular" (Denoiser.js:56-64)
            params = self._compose_params(cam_u)
            if self.isDebug:  # ssgi_compose.frag:21-24: the view itself, with its own sampler
                params = params or abi.SsgiComposeParams()
                params.is_debug = 1
            self.ctx.ssgi_compose(self._scene.depth, self.outputTexture, scene_buf, self.composer.outputBuffer, params=params)  # K5 (mainImage of the effect)

    def _compose_params(self, cam_u):
        """scene.fog -> the fog uniforms of ssgi_compose.frag (src/ssgi/SSGIEffect.js:80-90, 404-412); fog = dict(color, near, far) or
        dict(color, density, isFogExp2=True) like three.js Fog / FogExp2"""
        fog = getattr(self._scene, "fog", None)
        if not fog:
            return None
        p = abi.SsgiComposeParams()
        p.use_fog, p.fog_exp2 = 1, int(bool(fog.get("isFogExp2", False)))
        p.fog_color[:] = [float(x) for x in fog.get("color", (1.0, 1.0, 1.0))]
        p.fog_near, p.fog_far, p.fog_density = float(fog.get("near", 1.0)), float(fog.get("far", 1000.0)), float(fog.get("density", 0.00025))
        p.camera_near, p.camera_far, p.perspective = float(cam_u["near"]), float(cam_u["far"]), 1
        return p

    def dispose(self):
        if self._chain is not None:
            self._chain.close()
            self._chain = None
        if self.gBufferDebugTarget is not None:
            self.gBufferDebugTarget.free()
            self.gBufferDebugTarget = None


class SSREffect(SSGIEffect):
    """src/ssgi/SSREffect.js:3-9"""

    def __init__(self, composer, scene, camera, options=None):
        super().__init__(composer, scene, camera, {**defaultSSGIOptions, **(options or {}), "mode": "ssr"})


# ---------------------------------------------------------------------------------------------------
def generateR2(count: int) -> list:
    """src/temporal-reproject/utils/QuasirandomGenerator.js:11-24 (JS doubles)"""
    g = 1.32471795724474602596090885447809  # plastic number
    a1, a2, base = 1.0 / g, 1.0 / (g * g), 1.1127756842787055
    return [[math.fmod(base + a1 * n, 1.0), math.fmod(base + a2 * n, 1.0)] for n in range(count)]


r2Sequence = [[a - 0.5, b - 0.5] for a, b in generateR2(256)]  # src/taa/TAAUtils.js:3


def jitter(width, height, camera, frame: int, jitterScale: float = 1.0):
    """src/taa/TAAUtils.js:5-11: sub-pixel view offset from the R2 sequence (a no-op for cameras without setViewOffset)"""
    x, y = r2Sequence[frame % len(r2Sequence)]
    if hasattr(camera, "setViewOffset"):
        camera.setViewOffset(width, height, x * jitterScale, y * jitterScale, width, height)


class TemporalReprojectPass:
    """new TemporalReprojectPass(scene, camera, velocityDepthNormalPass, texture, textureCount, options)
    (src/temporal-reproject/TemporalReprojectPass.js:38-225).  1-plane RGBA16F configuration (TRAA)."""

    needsSwap = False

    def __init__(self, scene, camera, velocityDepthNormalPass, texture, textureCount, options=None):
        if textureCount != 1:
            raise abi.RfxError("standalone TemporalReprojectPass supports textureCount == 1 (the 2-plane SSGI form runs inside SSGIEffect)")
        self._scene, self._camera, self.velocityDepthNormalPass = scene, camera, velocityDepthNormalPass
        self.options = {**defaultTemporalReprojectPassOptions, **(options or {})}
        self.inputTexture, self.textureCount = texture, textureCount
        self.ctx: engine.Context = texture.ctx
        self.keepData, self._prev, self.frame = 1.0, None, 0
        self.renderTarget = self.framebufferTexture = None
        self.setSize(texture.width, texture.height)

    def setSize(self, width, height):
        for p in (self.renderTarget, self.framebufferTexture):
            if p is not None:
                p.free()
        self.renderTarget = self.ctx.alloc(abi.FMT_RGBA16F, width, height)
        self.framebufferTexture = self.ctx.alloc(abi.FMT_RGBA16F, width, height)  # copyFramebufferToTexture history (:197-200)

    @property
    def texture(self):
        """renderTarget.texture[0]: the plane rendered by the most recent render() (TemporalReprojectPass.js:150-156)"""
        return self.renderTarget

    def reset(self):
        self.keepData = 0.0

    def jitter(self, jitterScale: float = 1.0):  # TemporalReprojectPass.js:216-220
        self.unjitter()
        jitter(self.renderTarget.width, self.renderTarget.height, self._camera, self.frame, jitterScale)

    def unjitter(self):  # :222-224
        if hasattr(self._camera, "clearViewOffset"):
            self._camera.clearViewOffset()

    def render(self, renderer=None):
        self.frame = (self.frame + 1) % 4096
        # the pass uploads the UN-jittered projection (camera.view disabled around updateProjectionMatrix, :168-186)
        cam_u = self._camera.unjittered_uniforms() if hasattr(self._camera, "unjittered_uniforms") else self._camera.uniforms()
        prev = self._prev or cam_u
        o, p = self.options, abi.TemporalParams()
        p.cam = abi.make_camera(cam_u)
        abi.set_f16(p.prev_view_matrix, prev["view_matrix"])
        abi.set_f16(p.prev_camera_matrix_world, prev["camera_matrix_world"])
        abi.set_f16(p.prev_projection, prev["projection"])
        abi.set_f16(p.prev_projection_inverse, prev["projection_inverse"])
        p.camera_pos[:] = [float(x) for x in cam_u["position"]]
        p.prev_camera_pos[:] = [float(x) for x in prev["position"]]
        p.max_blend, p.neighborhood_clamp_intensity = o["maxBlend"], o["neighborhoodClampIntensity"]
        p.keep_data, p.confidence_power = self.keepData, o["confidencePower"]
        p.full_accumulate = int(bool(o["fullAccumulate"]) and not _did_camera_move(cam_u, self._prev))
        p.texture_count, p.input_type, p.log_transform, p.history_linear = 1, abi.INPUT_DIFFUSE, int(bool(o["logTransform"])), 1
        p.reproject_specular[:] = [0, 0]
        # the reference copies the framebuffer into framebufferTexture after the draw (:197-200); here the two planes swap roles
        # BEFORE the launch instead, so that `renderTarget` / `texture` is always the plane this render() wrote
        self.renderTarget, self.framebufferTexture = self.framebufferTexture, self.renderTarget
        self.ctx.temporal_reproject(p, self.inputTexture, self.velocityDepthNormalPass.texture, self.framebufferTexture, None, self.renderTarget, None)
        self.keepData = 1.0
        self._prev = cam_u

    @property
    def accumulated(self):
        return self.renderTarget

    def dispose(self):
        for p in (self.renderTarget, self.framebufferTexture):
            if p is not None:
                p.free()


class TRAAEffect:
    """new TRAAEffect(scene, camera, velocityDepthNormalPass, options)  (src/traa/TRAAEffect.js:10-76)"""

    DefaultOptions = defaultTemporalReprojectPassOptions

    def __init__(self, scene, camera, velocityDepthNormalPass, options=None):
        self._scene, self._camera, self.velocityDepthNormalPass = scene, camera, velocityDepthNormalPass
        forced = dict(maxBlend=0.9, neighborhoodClamp=True, neighborhoodClampIntensity=1, neighborhoodClampRadius=1, logTransform=True, confidencePower=4)
        self.options = {**defaultTemporalReprojectPassOptions, **(options or {}), **forced}  # :21-33
        self.temporalReprojectPass = None

    def setSize(self, width, height):
        if self.temporalReprojectPass:
            self.temporalReprojectPass.setSize(width, height)

    def reset(self):
        self.temporalReprojectPass.reset()

    def update(self, renderer=None, inputBuffer=None, deltaTime=None):
        if self.temporalReprojectPass is None:
            self.temporalReprojectPass = TemporalReprojectPass(self._scene, self._camera, self.velocityDepthNormalPass, inputBuffer, 1, self.options)
        self.temporalReprojectPass.inputTexture = inputBuffer
        trp = self.temporalReprojectPass
        trp.unjitter()                                                       # TRAAEffect.js:67-72
        self.unjitteredProjectionMatrix = np.array(getattr(self._camera, "proj", np.eye(4)), copy=True)
        trp.jitter()                                                         # the NEXT scene render is rasterised with this sub-pixel offset
        trp.render(renderer)

    def compose(self, outputBuffer):
        """traa_compose.frag: rgb passthrough, alpha 1"""
        self.temporalReprojectPass.ctx.traa_compose(self.temporalReprojectPass.accumulated, outputBuffer)

    def dispose(self):
        if self.temporalReprojectPass:
            self.temporalReprojectPass.dispose()


# ---------------------------------------------------------------------------------------------------
class PoissonDenoisePass:
    """new PoissonDenoisePass(camera, textures, options)  (src/denoise/pass/PoissonDenoisePass.js:26-150)"""

    DefaultOptions = defaultPoissonBlurOptions

    def __init__(self, camera, textures, options=None):
        o = {**defaultPoissonBlurOptions, **(options or {})}
        self.options, self.textures, self.iterations = o, list(textures), o["iterations"]
        self.ctx: engine.Context = self.textures[0].ctx
        self.textureCount = 2 if o["inputType"] == "diffuseSpecular" else 1
        self.isTextureSpecular = {"diffuseSpecular": [0, 1], "diffuse": [0, 0], "specular": [1, 1]}[o["inputType"]]
        self.radius, self.phi, self.lumaPhi, self.depthPhi, self.normalPhi = o["radius"], o["phi"], o["lumaPhi"], o["depthPhi"], o["normalPhi"]
        self.roughnessPhi, self.specularPhi = o.get("roughnessPhi", 0.0), o.get("specularPhi", 0.0)
        self._gbuffer = self._depth = None
        self._is_gbuffer = False
        self.blueNoiseIndex = BlueNoiseIndex(o.get("blueNoiseStart", 1234567))
        self.renderTargetA = self.renderTargetB = None
        self.setSize(self.textures[0].width, self.textures[0].height)

    def setSize(self, width, height):
        self.dispose()
        self.renderTargetA = [self.ctx.alloc(abi.FMT_RGBA16F, width, height) for _ in range(self.textureCount)]
        self.renderTargetB = [self.ctx.alloc(abi.FMT_RGBA16F, width, height) for _ in range(self.textureCount)]

    @property
    def texture(self):
        return self.renderTargetB

    def setGBufferPass(self, gbuffer_plane, depth_plane, is_gbuffer=True):
        """GBufferPass => GBUFFER_TEXTURE; VelocityDepthNormalPass => velocity-layout normals (:109-118)"""
        self._gbuffer, self._depth, self._is_gbuffer = gbuffer_plane, depth_plane, bool(is_gbuffer)

    def render(self, renderer=None):
        for i in range(2 * self.iterations):
            horizontal = i % 2 == 0
            src = self.textures if i == 0 else (self.renderTargetB if horizontal else self.renderTargetA)
            dst = self.renderTargetA if horizontal else self.renderTargetB
            p = abi.PoissonParams()
            p.radius, p.phi, p.luma_phi, p.depth_phi, p.normal_phi = self.radius, self.phi, self.lumaPhi, self.depthPhi, self.normalPhi
            p.roughness_phi, p.specular_phi = self.roughnessPhi, self.specularPhi
            p.texture_count = self.textureCount
            p.is_texture_specular[:] = self.isTextureSpecular
            p.gbuffer_texture = int(self._is_gbuffer)
            p.input_linear = int(i > 0 or src[0].format == abi.FMT_RGBA16F)
            p.blue_noise_index = self.blueNoiseIndex.value
            two = self.textureCount == 2
            self.ctx.poisson_denoise(p, self._depth, self._gbuffer, src[0], src[1] if two else None, dst[0], dst[1] if two else None)

    def dispose(self):
        for rt in (self.renderTargetA, self.renderTargetB):
            for p in rt or []:
                p.free()
        self.renderTargetA = self.renderTargetB = None


# ---------------------------------------------------------------------------------------------------
class HBAOEffect(_Reactive):
    """new HBAOEffect(composer, camera, scene, options)  (src/hbao/HBAOEffect.js:5-20, src/ao/AOEffect.js:23-178).
    The reference class does not compile at its pinned commit (SURVEY.md D3); this is hbao.frag + the 1-plane
    velocity-layout Poisson denoise + ao_compose.frag, the wiring the shaders are written for.

    resolutionScale (0, 1]: the AO pass renders to (int)(width * scale) x (int)(height * scale); the denoiser and the compose stay at
    full size and upsample it LINEAR (AOEffect.setSize :126-146).  normalTexture (an RGBA8 view-space normal plane) or useNormalPass
    (the host's NormalPass output, `scene.normal`) replaces the normal K6 rebuilds from depth; like the reference this is chosen at
    construction (:48-55)."""

    DefaultOptions = defaultAOOptions

    def __init__(self, composer, camera, scene, options=None):
        self.composer, self._camera, self._scene = composer, camera, scene
        self.ctx: engine.Context = composer.ctx
        self.blueNoiseIndex = BlueNoiseIndex((options or {}).get("blueNoiseStart", 1234567))
        o = {**defaultAOOptions, **(options or {})}
        o.pop("blueNoiseStart", None)
        _check_ao_scale(o["resolutionScale"])
        self._normal = o["normalTexture"]
        if self._normal is None and o["useNormalPass"]:
            self._normal = getattr(scene, "normal", None)
            if self._normal is None:
                raise abi.RfxError("HBAOEffect: useNormalPass needs the host's NormalPass output as scene.normal (RGBA8 view-space normals)")
        if self._normal is not None and self._normal.format != abi.FMT_RGBA8:
            raise abi.RfxError("HBAOEffect: the normal texture must be an RGBA8 plane (NormalPass layout)")
        self.aoTarget = self.ctx.alloc(abi.FMT_RGBA16F, composer.width, composer.height)
        self.PoissonDenoisePass = PoissonDenoisePass(camera, [self.aoTarget], dict(iterations=o["iterations"], radius=o["radius"], phi=o["phi"],
                                                                                    lumaPhi=o["lumaPhi"], depthPhi=o["depthPhi"],
                                                                                    normalPhi=o["normalPhi"], inputType="diffuse"))
        self._options = o
        self._resolution = (0.0, 0.0)  # {0, 0}: the AO target's own size
        self._lastSize = (composer.width, composer.height, 1)
        self.setSize(composer.width, composer.height)

    def __setattr__(self, k, v):
        if k == "resolutionScale":
            _check_ao_scale(v)
        super().__setattr__(k, v)

    def setSize(self, width, height):
        """AOEffect.setSize: a no-op when the size and the scale are unchanged; the AO target gets (int)(width * scale) x
        (int)(height * scale) and the unrounded product as its `resolution` (AOPass.js:79-83), the Poisson targets the full size"""
        s = self._options["resolutionScale"]
        if (width, height, s) == self._lastSize:
            return
        self.aoTarget.free()
        self.aoTarget = self.ctx.alloc(abi.FMT_RGBA16F, int(width * s), int(height * s))
        self._resolution = (width * s, height * s)
        self.PoissonDenoisePass.textures = [self.aoTarget]
        self.PoissonDenoisePass.setSize(width, height)
        self._lastSize = (width, height, s)

    def _option_changed(self, k):
        if k in ("iterations", "radius", "phi"):
            setattr(self.PoissonDenoisePass, k, self._options[k])
        elif k in ("lumaPhi", "depthPhi", "normalPhi"):
            setattr(self.PoissonDenoisePass, k, max(self._options[k], 0.0001))  # AOEffect.js:107-111
        elif k == "resolutionScale":
            self.setSize(*self._lastSize[:2])

    @property
    def texture(self):
        return self.PoissonDenoisePass.texture[0] if self._options["iterations"] > 0 else self.aoTarget

    def update(self, renderer=None, inputBuffer=None, deltaTime=None):
        o, cam_u = self._options, self._camera.uniforms()
        p = abi.HbaoParams()
        P = np.asarray(cam_u["projection"], np.float64).reshape(4, 4).T
        V = np.asarray(cam_u["view_matrix"], np.float64).reshape(4, 4).T
        abi.set_f16(p.projection_view, np.ascontiguousarray((P @ V).T.reshape(16)).astype(np.float32))  # AOPass.js:93-96
        abi.set_f16(p.projection_inverse, cam_u["projection_inverse"])
        abi.set_f16(p.camera_matrix_world, cam_u["camera_matrix_world"])
        abi.set_f16(p.view_matrix, cam_u["view_matrix"])
        p.resolution[:] = [float(self._resolution[0]), float(self._resolution[1])]
        p.ao_distance, p.distance_power, p.bias, p.thickness = o["distance"], o["distancePower"], o["bias"], o["thickness"]
        p.spp, p.blue_noise_index = int(o["spp"]), self.blueNoiseIndex.value
        self.ctx.hbao(p, self._scene.depth, self.aoTarget, normal=self._normal)
        self.PoissonDenoisePass.setGBufferPass(self._scene.velocity, self._scene.depth, is_gbuffer=False)
        self.PoissonDenoisePass.render(renderer)
        if inputBuffer is not None and getattr(self.composer, "outputBuffer", None) is not None:
            c = abi.AoComposeParams()
            c.power = o["power"]
            c.color[:] = [float(x) for x in o["color"]]
            self.ctx.ao_compose(c, self._scene.depth, self.texture, inputBuffer, self.composer.outputBuffer)

    def dispose(self):
        self.PoissonDenoisePass.dispose()
        self.aoTarget.free()


def _check_ao_scale(s):
    if not (isinstance(s, (int, float)) and 0.0 < s <= 1.0):
        raise abi.RfxError(f"HBAOEffect: resolutionScale must lie in (0, 1], got {s!r}")


# ---------------------------------------------------------------------------------------------------
# HorizonAOEffect: AOEffect's keys that still mean something for a horizon march, plus the march's own; spp, distancePower, bias and
# thickness (read only by hbao.frag's hemisphere samples) are not carried.
defaultHorizonAOOptions = dict(
    resolutionScale=1, distance=2, power=2, color=(0.0, 0.0, 0.0), useNormalPass=False, velocityDepthNormalPass=None, normalTexture=None,
    directions=8, steps=32, angleBias=0.1, intensity=1, maxRadiusPixels=64, **defaultPoissonBlurOptions)

_HORIZON_RANGES = {  # key: (test, what the error says)
    "directions": (lambda v: isinstance(v, int) and 1 <= v <= 32, "an integer in 1..32"),
    "steps": (lambda v: isinstance(v, int) and 1 <= v <= 64, "an integer in 1..64"),
    "distance": (lambda v: math.isfinite(v) and v > 0, "> 0"),
    "angleBias": (lambda v: 0 <= v < 1, "in [0, 1)"),
    "intensity": (lambda v: math.isfinite(v) and v >= 0, ">= 0"),
    "maxRadiusPixels": (lambda v: v >= 1, ">= 1"),
}


def check_horizon_ao_options(o: dict) -> None:
    """HorizonAOEffect's option ranges (those rfx_hbao_horizon_launch enforces, and resolutionScale in (0, 1]); raises abi.RfxError"""
    _check_ao_scale(o["resolutionScale"])
    for k, (ok, what) in _HORIZON_RANGES.items():
        v = o[k]
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not ok(v):
            raise abi.RfxError(f"HorizonAOEffect: {k} must be {what}, got {v!r}")


class HorizonAOEffect(HBAOEffect):
    """new HorizonAOEffect(composer, camera, scene, options): HBAOEffect with K6h, the horizon march (directions x steps depth taps per
    pixel; DESIGN.md §1 K6h), in place of hbao.frag.  An extension: the reference has no such effect (SURVEY.md D1).  The AO target and
    its resolutionScale, the normal plane (useNormalPass / normalTexture), the one-plane Poisson denoise and ao_compose are HBAOEffect's.
    Options are reactive and range-checked before any launch."""

    DefaultOptions = defaultHorizonAOOptions

    def __init__(self, composer, camera, scene, options=None):
        o = {**defaultHorizonAOOptions, **(options or {})}
        check_horizon_ao_options(o)
        super().__init__(composer, camera, scene, o)
        for k in ("spp", "distancePower", "bias", "thickness"):  # HBAOEffect's hemisphere-sample keys: not options of this effect
            if k not in o:
                del self._options[k]

    def __setattr__(self, k, v):
        o = self.__dict__.get("_options")
        if o is not None and k in _HORIZON_RANGES:
            check_horizon_ao_options({**o, k: v})
        super().__setattr__(k, v)

    def update(self, renderer=None, inputBuffer=None, deltaTime=None):
        o, cam_u = self._options, self._camera.uniforms()
        p = abi.HbaoHorizonParams()
        for k in ("projection", "projection_inverse", "camera_matrix_world", "view_matrix"):
            abi.set_f16(getattr(p, k), cam_u[k])
        p.resolution[:] = [float(self._resolution[0]), float(self._resolution[1])]
        p.distance, p.angle_bias, p.intensity, p.max_radius_pixels = o["distance"], o["angleBias"], o["intensity"], o["maxRadiusPixels"]
        p.directions, p.steps, p.blue_noise_index = int(o["directions"]), int(o["steps"]), self.blueNoiseIndex.value
        self.ctx.hbao_horizon(p, self._scene.depth, self.aoTarget, normal=self._normal)
        self.PoissonDenoisePass.setGBufferPass(self._scene.velocity, self._scene.depth, is_gbuffer=False)
        self.PoissonDenoisePass.render(renderer)
        if inputBuffer is not None and getattr(self.composer, "outputBuffer", None) is not None:
            c = abi.AoComposeParams()
            c.power = o["power"]
            c.color[:] = [float(x) for x in o["color"]]
            self.ctx.ao_compose(c, self._scene.depth, self.texture, inputBuffer, self.composer.outputBuffer)


# ---------------------------------------------------------------------------------------------------
class MotionBlurEffect(_Reactive):
    """new MotionBlurEffect(velocityPass, options)  (src/motion-blur/MotionBlurEffect.js:16-102)"""

    def __init__(self, velocityPass, options=None):
        self.velocityPass = velocityPass
        self._frame = 0
        self._options = {**defaultMotionBlurOptions, **(options or {})}

    def update(self, renderer=None, inputBuffer=None, deltaTime=1 / 60, outputBuffer=None, window=None):
        """window = (innerWidth, innerHeight): the reference feeds the CSS window size as `resolution` (A10)."""
        ctx: engine.Context = inputBuffer.ctx
        p = abi.MotionBlurParams()
        p.intensity, p.jitter = self._options["intensity"], self._options["jitter"]
        p.delta_time = max(1 / 1000, deltaTime)
        p.resolution[:] = list(window or (inputBuffer.width, inputBuffer.height))
        p.frame = self._frame % 4096  # renderer.info.render.frame % 4096
        p.samples = int(self._options["samples"])
        self._frame += 1
        ctx.motion_blur(p, self.velocityPass.texture, inputBuffer, outputBuffer)


def getMaxMipLevel(width: int, height: int) -> int:
    """src/ssgi/utils/Utils.js:30-34"""
    return math.floor(math.log2(max(width, height))) + 1


# ---------------------------------------------------------------------------------------------------
# Cosmetic effects of the plugin surface (src/index.js:25-31) and the pass that merges them.
# ---------------------------------------------------------------------------------------------------
class SharpnessEffect:
    """new SharpnessEffect(options)  (src/sharpness/SharpnessEffect.js:36-59)"""

    fx_id = abi.FX_SHARPNESS

    def __init__(self, options=None):
        self.sharpness = {"sharpness": 1, **(options or {})}["sharpness"]

    def setSharpness(self, sharpness):
        self.sharpness = sharpness

    def update(self, renderer=None, inputBuffer=None, deltaTime=None):
        pass  # `inputTexture = inputBuffer.texture`: the merged kernel reads the pass input directly

    def _fill(self, p: abi.EffectsParams):
        p.sharpness = float(self.sharpness)


class LensDistortionEffect:
    """new LensDistortionEffect({ alphax, alphay, aberration })  (src/lens-distortion/LensDistortionEffect.js:48-77)"""

    fx_id = abi.FX_LENS_DISTORTION

    def __init__(self, options=None):
        o = {"alphax": -0.05, "alphay": -0.05, "aberration": 1, **(options or {})}
        self.alphax, self.alphay, self.aberration = o["alphax"], o["alphay"], o["aberration"]

    def setAlphaX(self, value):
        self.alphax = value

    def setAlphaY(self, value):
        self.alphay = value

    def update(self, renderer=None, inputBuffer=None, deltaTime=None):
        pass

    def _fill(self, p: abi.EffectsParams):
        p.alphax, p.alphay, p.aberration = float(self.alphax), float(self.alphay), float(self.aberration)


class GradualBackgroundEffect:
    """new GradualBackgroundEffect(camera, depthTexture, backgroundColor, maxDistance = 5)  (src/gradual-background/GradualBackgroundEffect.js:48-70)"""

    fx_id = abi.FX_GRADUAL_BACKGROUND

    def __init__(self, camera, depthTexture, backgroundColor, maxDistance=5):
        self._camera, self.depthTexture, self.backgroundColor, self.maxDistance = camera, depthTexture, tuple(backgroundColor), maxDistance

    def setBackgroundColor(self, color):
        self.backgroundColor = tuple(color)

    def setMaxDistance(self, distance):
        self.maxDistance = distance

    def update(self, renderer=None, inputBuffer=None, deltaTime=None):
        pass

    def _fill(self, p: abi.EffectsParams):
        p.background_color[:] = [float(c) for c in self.backgroundColor]
        p.max_distance = float(self.maxDistance)


class SparkleEffect:
    """new SparkleEffect(camera, velocityDepthNormalPass)  (src/sparkle/SparkleEffect.js:102-136).  The reference never defines
    PERSPECTIVE_CAMERA for this effect, so its getViewZ takes the orthographic branch; `definePerspectiveCamera = True` gives what a host
    that defines it gets."""

    fx_id = abi.FX_SPARKLE

    def __init__(self, camera, velocityDepthNormalPass, definePerspectiveCamera=False):
        self._camera, self.velocityDepthNormalPass = camera, velocityDepthNormalPass
        self.spread, self.intensity, self.definePerspectiveCamera = 1, 1, definePerspectiveCamera

    def setSpread(self, spread):
        self.spread = spread

    def setIntensity(self, intensity):
        self.intensity = intensity

    def update(self, renderer=None, inputBuffer=None, deltaTime=None):
        pass

    def _fill(self, p: abi.EffectsParams):
        p.spread, p.intensity, p.sparkle_perspective = float(self.spread), float(self.intensity), int(bool(self.definePerspectiveCamera))


class EffectPass:
    """postprocessing's `new EffectPass(camera, ...effects)` for the four effects above: the effects of one pass are merged into one
    fullscreen program — here ONE launch of rfx_effects_launch (csrc/k_fx.cu) — in which every effect samples the pass's input buffer
    and the colour flows from one effect to the next in the given order."""

    def __init__(self, camera, *effects):
        if not 1 <= len(effects) <= 4:
            raise ValueError("EffectPass: 1..4 effects")
        self._camera, self.effects = camera, list(effects)

    def render(self, renderer, inputBuffer, outputBuffer, deltaTime=None, stencilTest=None):
        ctx: engine.Context = inputBuffer.ctx
        p = abi.make_effects_params(self._camera.uniforms(), [e.fx_id for e in self.effects])
        depth = velocity = None
        for e in self.effects:
            e.update(renderer, inputBuffer, deltaTime)
            e._fill(p)
            if isinstance(e, GradualBackgroundEffect):
                depth = e.depthTexture
            if isinstance(e, SparkleEffect):
                velocity = e.velocityDepthNormalPass.texture
        ctx.effects(p, inputBuffer, depth, velocity, outputBuffer)


class TAAPass:
    """new TAAPass(camera)  (src/taa/TAAPass.js:18-95): the still-camera accumulator that renders to the screen.  `canvas` (RGBA8) stands in
    for the default framebuffer; the FramebufferTexture copy of it is the history.  `srgbOutput` = the renderer's output colour space."""

    renderToScreen = True

    def __init__(self, camera, srgbOutput=True):
        self._camera, self.srgbOutput = camera, srgbOutput
        self.cameraNotMovedFrames, self.frame, self.needsUpdate = 0, 0, False
        self._last = None
        self.canvas = self.framebufferTexture = None

    def setSize(self, width, height, ctx: "engine.Context | None" = None):
        """setSize(width, height) as in the reference (:57-66); the planes are allocated on `ctx`, or on the input buffer's context at the next render()"""
        self.dispose()
        self._size, self.needsUpdate = (int(width), int(height)), True
        if ctx is not None:
            self.canvas = ctx.alloc(abi.FMT_RGBA8, width, height)
            self.framebufferTexture = ctx.alloc(abi.FMT_RGBA8, width, height)

    def render(self, renderer, inputBuffer):
        ctx: engine.Context = inputBuffer.ctx
        if self.canvas is None:
            w, h = getattr(self, "_size", (inputBuffer.width, inputBuffer.height))
            self.canvas, self.framebufferTexture = ctx.alloc(abi.FMT_RGBA8, w, h), ctx.alloc(abi.FMT_RGBA8, w, h)
        self.frame = (self.frame + 1) % 4096
        cam_u = self._camera.uniforms()
        moved = self.needsUpdate or _did_camera_move(cam_u, self._last)
        self.needsUpdate = False
        n = self.cameraNotMovedFrames
        if n > 0:  # :81-84
            jitter(self.canvas.p.width, self.canvas.p.height, self._camera, self.frame, 1)
        self.cameraNotMovedFrames = 0 if moved else (n + 1) % 4096
        self._last = cam_u
        p = abi.TaaParams()
        p.camera_not_moved_frames, p.srgb_output = float(self.cameraNotMovedFrames), int(bool(self.srgbOutput))
        ctx.taa(p, inputBuffer, self.framebufferTexture, self.canvas)
        self.framebufferTexture, self.canvas = self.canvas, self.framebufferTexture  # copyFramebufferToTexture (:93): the canvas becomes the history
        return self.framebufferTexture

    def dispose(self):
        for pl in (self.canvas, self.framebufferTexture):
            if pl is not None:
                pl.free()
        self.canvas = self.framebufferTexture = None
