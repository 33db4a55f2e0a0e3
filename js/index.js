// js/index.js — the reference's plugin surface (src/index.js:16-31) over the N-API shim (js/napi/shim.cc).
//
// NOT RUNNABLE IN THIS IMAGE (no Node, no GL; SURVEY.md D5) — this is the reference-side glue a maintainer adds to drop the
// CUDA engine under a postprocessing.js EffectComposer: the reference's eight classes with its constructor signatures, option
// names / defaults, reactive option properties and `update(renderer, inputBuffer, deltaTime)` / `render(renderer)` /
// `setSize` / `initialize` / `reset` / `dispose` methods.  The tested host mirror of the same surface is
// realism_effects_b200/effects.py (each method there ends in the same rfx_* entry point this file reaches through the shim).
//
// Plane transport: three.js keeps rasterising the G-buffer / velocity / scene-colour render targets (SURVEY.md K10/K11: out of
// scope as compute).  A `PlaneSource` turns them into device planes for the engine; the default one reads the render targets
// back (renderer.readRenderTargetPixels -> typed arrays -> rfx.planeUpload).  The zero-copy variant (cudaGraphicsGLRegisterImage
// on the WebGL textures) is SURVEY.md §8(f) row 4 and replaces only this class.
import { createRequire } from "node:module"
const rfx = createRequire(import.meta.url)("./napi/rfx_napi.node")

const FMT = { R32F: 0, RGBA32F: 1, RGBA16F: 2, RGBA8: 3 }
const FLAG = { importanceSampling: 1, missedRays: 2, useDirectLight: 4, useEnvMap: 8 }
const INPUT = { diffuseSpecular: 0, diffuse: 1, specular: 2 }
// rfx_ssgi_chain_set_debug_view (include/rfx.h): chain output n is output + n, GBufferDebugPass mode m gbufferChannel + m
export const DEBUG_VIEW = { none: -1, output: 0, depth: 8, velocity: 9, gbuffer: 10, gbufferChannel: 16 }
export const GBUFFER_DEBUG_MODES = ["diffuse", "alpha", "normal", "roughness", "metalness", "emissive"]   // SSGIEffect.js:237
let sharedCtx = null
export const context = (device = 0) => (sharedCtx ??= rfx.ctxCreate(device))

const f32 = m => new Float32Array(m.elements ?? m)
const cameraBlock = camera => ({
	projection: f32(camera.projectionMatrix), projectionInverse: f32(camera.projectionMatrixInverse),
	matrixWorld: f32(camera.matrixWorld), matrixWorldInverse: f32(camera.matrixWorldInverse), near: camera.near, far: camera.far,
	perspective: camera.isPerspectiveCamera !== false
})
// src/utils/SceneUtils.js:17-27
const didCameraMove = (camera, lastPos, lastQuat) =>
	!lastPos || camera.position.distanceToSquared(lastPos) > 1e-6 || 8 * (1 - lastQuat.dot(camera.quaternion)) > 1e-6

// src/utils/BlueNoiseUtils.js:17-33 — one closure per material; the index advances on every uniform READ
class BlueNoiseIndex {
	constructor(start = Math.floor(Math.random() * 65536)) { this.start = start; this.index = 0 }
	get value() { this.index = (this.start + this.index + 1) % 0x7fffffff; return this.index }
}

const reactive = (self, options, onChange) => {
	for (const key of Object.keys(options)) {
		Object.defineProperty(self, key, {
			get: () => options[key],
			set: value => { if (options[key] === value) return; options[key] = value; onChange(key, value) },
			configurable: true
		})
	}
}

// Default PlaneSource: read the three.js render targets back and upload them.  planes: { depth, gbuffer, velocity, directLight }
export class ReadbackPlaneSource {
	constructor(ctx, width, height) { this.ctx = ctx; this.resize(width, height) }
	resize(width, height) {
		this.dispose()
		this.width = width; this.height = height
		const n = width * height
		this.host = { depth: new Float32Array(n), gbuffer: new Float32Array(4 * n), velocity: new Float32Array(4 * n), directLight: new Uint16Array(4 * n) }
		this.dev = { depth: rfx.planeAlloc(this.ctx, FMT.R32F, width, height), gbuffer: rfx.planeAlloc(this.ctx, FMT.RGBA32F, width, height),
			velocity: rfx.planeAlloc(this.ctx, FMT.RGBA32F, width, height), directLight: rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height) }
	}
	// targets: { depth: WebGLRenderTarget (R32F copy of the depth texture), gbuffer, velocity, directLight }
	read(renderer, targets) {
		for (const k of Object.keys(this.dev)) {
			if (!targets[k]) continue
			renderer.readRenderTargetPixels(targets[k], 0, 0, this.width, this.height, this.host[k])
			rfx.planeUpload(this.ctx, this.dev[k], this.host[k])
		}
		return this.dev
	}
	dispose() { if (this.dev) for (const p of Object.values(this.dev)) rfx.planeFree(this.ctx, p); this.dev = null }
}

// PlaneSource for hosts WITHOUT the reference's rasteriser materials (GBufferMaterial / VelocityDepthNormalMaterial): upload a
// conventional deferred renderer's planes and let the GPU pack them (rfx_gbuffer_ingest_launch = packGBuffer, gbuffer_packing.glsl:166-178,
// + the velocity layout of VelocityDepthNormalMaterial.js:76-83,186-188).  host: { albedo: Uint8Array RGBA8, normal: Uint16Array RGBA16F
// (world space), material: Uint8Array RGBA8 (r roughness, g metalness), emissive: Uint16Array RGBA16F | null, motion: Uint16Array RGBA16F
// (uv-space cur - prev) | null, depth: Float32Array, directLight: Uint16Array RGBA16F }
export class IngestPlaneSource {
	constructor(ctx, width, height, { motionScale = [1, 1], normalizeNormals = true } = {}) { this.ctx = ctx; this.opt = { motionScale, normalizeNormals: normalizeNormals ? 1 : 0 }; this.resize(width, height) }
	resize(width, height) {
		this.dispose()
		this.width = width; this.height = height
		const a = fmt => rfx.planeAlloc(this.ctx, fmt, width, height)
		this.src = { albedo: a(FMT.RGBA8), normal: a(FMT.RGBA16F), material: a(FMT.RGBA8), emissive: a(FMT.RGBA16F), motion: a(FMT.RGBA16F) }
		this.dev = { depth: a(FMT.R32F), gbuffer: a(FMT.RGBA32F), velocity: a(FMT.RGBA32F), directLight: a(FMT.RGBA16F) }
	}
	read(_renderer, host) {
		for (const k of Object.keys(this.src)) if (host[k]) rfx.planeUpload(this.ctx, this.src[k], host[k])
		rfx.planeUpload(this.ctx, this.dev.depth, host.depth)
		if (host.directLight) rfx.planeUpload(this.ctx, this.dev.directLight, host.directLight)
		rfx.gbufferIngest(this.ctx, this.opt, this.src.albedo, this.src.normal, this.src.material, host.emissive ? this.src.emissive : null,
			host.motion ? this.src.motion : null, this.dev.depth, this.dev.gbuffer, this.dev.velocity)
		return this.dev
	}
	dispose() { for (const set of [this.src, this.dev]) if (set) for (const p of Object.values(set)) rfx.planeFree(this.ctx, p); this.src = this.dev = null }
}

// -------------------------------------------------------------------------------------------------------------------------
export class VelocityDepthNormalPass {
	// new VelocityDepthNormalPass(scene, camera) — src/temporal-reproject/pass/VelocityDepthNormalPass.js:71-91.
	// Rasterisation stays in three.js (`rasterPass`: the reference's own pass object); this wrapper exposes what others read.
	constructor(scene, camera, rasterPass) { this._scene = scene; this._camera = camera; this.rasterPass = rasterPass; this.needsSwap = false }
	get texture() { return this.rasterPass.texture }
	get renderTarget() { return this.rasterPass.renderTarget }
	get lastVelocityTexture() { return this.rasterPass.lastVelocityTexture }
	setSize(w, h) { this.rasterPass.setSize(w, h) }
	render(renderer) { this.rasterPass.render(renderer) }
	dispose() { this.rasterPass.dispose() }
}

// src/temporal-reproject/pass/VelocityPass.js:3-7 — the same pass with the depth / normal outputs switched off
export class VelocityPass extends VelocityDepthNormalPass {
	constructor(scene, camera, rasterPass) { super(scene, camera, rasterPass) }
}

// src/ssgi/SSGIOptions.js:26-48
export const defaultSSGIOptions = {
	mode: "ssgi", distance: 10, thickness: 10, denoiseIterations: 1, denoiseKernel: 2, denoiseDiffuse: 10, denoiseSpecular: 10,
	radius: 3, phi: 0.5, lumaPhi: 5, depthPhi: 2, normalPhi: 50, roughnessPhi: 50, specularPhi: 50, envBlur: 0.5,
	importanceSampling: true, steps: 20, refineSteps: 5, resolutionScale: 1, missedRays: false, outputTexture: null
}

export class SSGIEffect {
	// new SSGIEffect(composer, scene, camera, options) — src/ssgi/SSGIEffect.js:31 (the code's signature, SURVEY.md D6)
	constructor(composer, scene, camera, options = {}) {
		this.composer = composer; this._scene = scene; this._camera = camera
		const opts = { denoiseMode: "full", ...defaultSSGIOptions, ...options }
		if (typeof opts.preset === "string") {   // src/ssgi/SSGIEffect.js:79-99
			if (opts.preset === "low") Object.assign(opts, { steps: 10, refineSteps: 2, denoiseMode: "full_temporal" })
			else if (opts.preset === "medium") Object.assign(opts, { steps: 20, refineSteps: 4, denoiseMode: "full" })
		}
		this._options = opts
		this.ctx = context(options.device ?? 0)
		this.velocityDepthNormalPass = options.velocityDepthNormalPass
		this.gBufferPass = options.gBufferPass                       // three.js GBufferPass: { texture, depthTexture, renderTarget }
		this.isUsingRenderPass = true
		this._hasEnv = false
		this.lastPos = null; this.lastQuat = null
		// textures a debug view can name that outlive setSize: chain output n (the fast chain re-splits trOut / dnB when read) and the
		// frame's planes of the plane source; denoiserTexture is chain output 0, denoiser.texture (Denoiser.js:67-78)
		this._chainTextures = [0, 1, 2, 3, 4, 5].map(n => ({ chainOutput: n }))
		this._frameTextures = { depth: { framePlane: "depth" }, velocity: { framePlane: "velocity" }, gbuffer: { framePlane: "gbuffer" } }
		this.denoiserTexture = this._chainTextures[0]
		this._view = null; this.isDebug = false; this.gBufferDebugTarget = null; this._gBufferDebugMode = 0
		reactive(this, opts, key => (key === "resolutionScale" ? this.setSize(this.width, this.height, true) : this._setOptions()))
		// outputTexture (SSGIEffect.js:228-251): not a chain option and no reset()
		Object.defineProperty(this, "outputTexture", { get: () => this._view ?? this.denoiserTexture, set: v => this._setOutputTexture(v), configurable: true })
		opts.outputTexture = this.denoiserTexture   // :139
		this.setSize(options.width ?? composer?.inputBuffer?.width, options.height ?? composer?.inputBuffer?.height)
	}
	chainTexture(n) { return this._chainTextures[n] }            // chain output n (1 ssgiOut, 2/3 trOut, 4/5 dnB) as a debug view
	frameTexture(name) { return this._frameTextures[name] }      // "depth" | "velocity" | "gbuffer": the frame's plane as a debug view
	// falsy: ignored; a string: GBufferDebugPass mode (index in GBUFFER_DEBUG_MODES, -1 = emissive) rendered after the chain, whose target
	// becomes the view; a texture (chainTexture / frameTexture / a plane the host holds): that texture.  isDebug = view !== denoiserTexture
	_setOutputTexture(value) {
		if (!value) return
		if (typeof value === "string") {
			this.gBufferDebugTarget ??= rfx.planeAlloc(this.ctx, FMT.RGBA32F, this.width, this.height)
			this._gBufferDebugMode = GBUFFER_DEBUG_MODES.indexOf(value)
			this._view = this.gBufferDebugTarget
		} else {
			if (this.gBufferDebugTarget && value !== this.gBufferDebugTarget) { rfx.planeFree(this.ctx, this.gBufferDebugTarget); this.gBufferDebugTarget = null }
			this._view = value === this.denoiserTexture ? null : value
		}
		this.isDebug = this._view !== null
		this._options.outputTexture = this.outputTexture
	}
	_resolve(t, planes) {
		if (t.chainOutput !== undefined) return rfx.chainOutput(this.ctx, this.chain, t.chainOutput)
		if (t.framePlane !== undefined) return planes[t.framePlane]
		return t
	}
	_flags() {
		const o = this._options
		return (o.importanceSampling && this._hasEnv ? FLAG.importanceSampling : 0) | (o.missedRays ? FLAG.missedRays : 0) |
			(this.isUsingRenderPass ? FLAG.useDirectLight : 0) | (this._hasEnv ? FLAG.useEnvMap : 0)
	}
	_chainOptions() {
		const denoiseModeId = ["full", "full_temporal", "temporal"].indexOf(this._options.denoiseMode ?? "full")   // Denoiser.js:7
		if (denoiseModeId < 0) throw new Error(`denoiseMode "${this._options.denoiseMode}" cannot run (in the reference "denoised" binds an array of textures to a sampler)`)
		return { ...this._options, width: this.width, height: this.height, flags: this._flags(), mode: this._options.mode === "ssr" ? 1 : 0, denoiseModeId }
	}
	_setOptions() { if (this.chain) rfx.chainSetOptions(this.ctx, this.chain, this._chainOptions()) }   // setters end with reset() (SSGIEffect.js:203-209)
	setSize(width, height, force = false) {
		if (width === undefined || (!force && width === this.width && height === this.height)) return
		this.width = width; this.height = height
		if (this.chain) rfx.chainDestroy(this.chain)
		this.chain = rfx.chainCreate(this.ctx, this._chainOptions())
		this.planeSource?.dispose()
		this.planeSource = new ReadbackPlaneSource(this.ctx, width, height)
		this.outputPlane = rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height)
		this.outputHost = new Uint16Array(width * height * 4)
		if (this.gBufferDebugTarget) {   // GBufferDebugPass.setSize at the effect's size
			rfx.planeFree(this.ctx, this.gBufferDebugTarget)
			this.gBufferDebugTarget = this._view = rfx.planeAlloc(this.ctx, FMT.RGBA32F, width, height)
		}
	}
	// keepEnvMapUpdated (src/ssgi/SSGIEffect.js:309-366): equirect RGBA16F map; the CDF tables are built on the device
	setEnvironment(mapF16, width, height) { rfx.envBuild(this.ctx, mapF16, width, height); this._hasEnv = true; this._setOptions() }
	clearEnvironment() { rfx.envClear(this.ctx); this._hasEnv = false; this._setOptions() }
	initialize() {}
	reset() { rfx.chainReset(this.chain) }
	get depthTexture() { return this.gBufferPass?.depthTexture }
	// outputHost: the K5 output (RGBA16F), uploaded into the composer's output buffer by the glue.  outputTexture: see the constructor.
	// update(renderer, inputBuffer, deltaTime) — src/ssgi/SSGIEffect.js:372-404
	update(renderer, inputBuffer, deltaTime) {
		const cam = cameraBlock(this._camera)
		const moved = didCameraMove(this._camera, this.lastPos, this.lastQuat)
		this.lastPos = this._camera.position.clone(); this.lastQuat = this._camera.quaternion.clone()
		this.velocityDepthNormalPass?.render(renderer)
		const planes = this.planeSource.read(renderer, { depth: this.gBufferPass?.depthRenderTarget, gbuffer: this.gBufferPass?.renderTarget,
			velocity: this.velocityDepthNormalPass?.renderTarget, directLight: inputBuffer })
		rfx.chainRender(this.ctx, this.chain, cam, planes.depth, planes.gbuffer, planes.velocity, this.isUsingRenderPass ? planes.directLight : null,
			new Float32Array(this._camera.position.toArray()), moved)
		if (this.gBufferDebugTarget) rfx.gbufferDebug(this.ctx, this._gBufferDebugMode, planes.gbuffer, this.gBufferDebugTarget)   // SSGIEffect.js:398-399
		// K5: ssgi_compose.frag (mainImage of the effect); with isDebug the view itself, with its own sampler (:21-24)
		const fog = this._scene.fog   // SSGIEffect.js:404-412
		rfx.ssgiCompose(this.ctx, planes.depth, this._resolve(this.outputTexture, planes), planes.directLight, this.outputPlane, {
			near: this._camera.near, far: this._camera.far, perspective: this._camera.isPerspectiveCamera !== false, isDebug: this.isDebug,
			...(fog ? { fog: { color: fog.color.toArray(), near: fog.near, far: fog.far, density: fog.density, isFogExp2: !!fog.isFogExp2 } } : {})
		})
		rfx.planeDownload(this.ctx, this.outputPlane, this.outputHost)
	}
	dispose() {
		if (this.chain) rfx.chainDestroy(this.chain)
		this.chain = null
		this.planeSource?.dispose()
		if (this.outputPlane) rfx.planeFree(this.ctx, this.outputPlane)
		if (this.gBufferDebugTarget) rfx.planeFree(this.ctx, this.gBufferDebugTarget)
		this.outputPlane = this.gBufferDebugTarget = null
	}
}
SSGIEffect.DefaultOptions = defaultSSGIOptions

export class SSREffect extends SSGIEffect {
	// src/ssgi/SSREffect.js:3-9
	constructor(composer, scene, camera, options = {}) { super(composer, scene, camera, { ...options, mode: "ssr" }) }
}

// -------------------------------------------------------------------------------------------------------------------------
// src/temporal-reproject/TemporalReprojectPass.js:17-32
export const defaultTemporalReprojectPassOptions = {
	dilation: false, fullAccumulate: false, neighborhoodClamp: false, neighborhoodClampRadius: 1, neighborhoodClampIntensity: 1, maxBlend: 1,
	logTransform: false, depthDistance: 2, worldDistance: 4, reprojectSpecular: false, renderTarget: null, copyTextures: true,
	confidencePower: 0.75, inputType: "diffuse"
}

// src/temporal-reproject/utils/QuasirandomGenerator.js:11-24, src/taa/TAAUtils.js:3-11
export const generateR2 = count => {
	const g = 1.32471795724474602596090885447809, a1 = 1.0 / g, a2 = 1.0 / (g * g), base = 1.1127756842787055
	return Array.from({ length: count }, (_, n) => [(base + a1 * n) % 1, (base + a2 * n) % 1])
}
export const r2Sequence = generateR2(256).map(([a, b]) => [a - 0.5, b - 0.5])
export function jitter(width, height, camera, frame, jitterScale = 1) {
	const [x, y] = r2Sequence[frame % r2Sequence.length]
	if (camera.setViewOffset) camera.setViewOffset(width, height, x * jitterScale, y * jitterScale, width, height)
}

export class TemporalReprojectPass {
	// new TemporalReprojectPass(scene, camera, velocityDepthNormalPass, texture, textureCount, options) — TemporalReprojectPass.js:38-225
	// (stand-alone 1-plane RGBA16F form, as TRAAEffect uses it; the 2-plane SSGI form runs inside the native chain)
	constructor(scene, camera, velocityDepthNormalPass, texture, textureCount = 1, options = defaultTemporalReprojectPassOptions) {
		if (textureCount !== 1) throw new Error("stand-alone TemporalReprojectPass: textureCount must be 1")
		this._scene = scene; this._camera = camera; this.velocityDepthNormalPass = velocityDepthNormalPass
		this.inputTexture = texture; this.textureCount = textureCount
		this.options = { ...defaultTemporalReprojectPassOptions, ...options }
		this.ctx = context(); this.needsSwap = false; this.frame = 0; this.keepData = 1; this.prev = null
		this.lastPos = null; this.lastQuat = null
	}
	setSize(width, height) {
		this.dispose()
		this.width = width; this.height = height
		this.renderTarget = rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height)
		this.framebufferTexture = rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height)   // copyFramebufferToTexture history (:197-200)
		this.inputPlane = rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height)
		this.velocityPlane = rfx.planeAlloc(this.ctx, FMT.RGBA32F, width, height)
		this.hostIn = new Uint16Array(4 * width * height); this.hostVel = new Float32Array(4 * width * height)
	}
	get texture() { return this.renderTarget }   // renderTarget.texture[0]: the plane the most recent render() wrote (:150-156)
	reset() { this.keepData = 0 }
	jitter(jitterScale = 1) { this.unjitter(); jitter(this.width, this.height, this._camera, this.frame, jitterScale) }
	unjitter() { if (this._camera.clearViewOffset) this._camera.clearViewOffset() }
	render(renderer) {
		this.frame = (this.frame + 1) % 4096
		// the pass uploads the UN-jittered projection (:168-186)
		const proj = this._camera.projectionMatrix.clone(), projInv = this._camera.projectionMatrixInverse.clone()
		if (this._camera.view) this._camera.view.enabled = false
		this._camera.updateProjectionMatrix()
		const cam = cameraBlock(this._camera)
		if (this._camera.view) this._camera.view.enabled = true
		this._camera.projectionMatrix.copy(proj); this._camera.projectionMatrixInverse.copy(projInv)
		const prev = this.prev ?? cam
		const full = this.options.fullAccumulate && !didCameraMove(this._camera, this.lastPos, this.lastQuat)
		this.lastPos = this._camera.position.clone(); this.lastQuat = this._camera.quaternion.clone()
		renderer.readRenderTargetPixels(this.inputTexture, 0, 0, this.width, this.height, this.hostIn)
		renderer.readRenderTargetPixels(this.velocityDepthNormalPass.renderTarget, 0, 0, this.width, this.height, this.hostVel)
		rfx.planeUpload(this.ctx, this.inputPlane, this.hostIn); rfx.planeUpload(this.ctx, this.velocityPlane, this.hostVel)
		;[this.renderTarget, this.framebufferTexture] = [this.framebufferTexture, this.renderTarget]   // the last result becomes the history
		rfx.temporalReproject(this.ctx, {
			cam, prev, cameraPos: new Float32Array(this._camera.position.toArray()), maxBlend: this.options.maxBlend,
			neighborhoodClampIntensity: this.options.neighborhoodClampIntensity, keepData: this.keepData, confidencePower: this.options.confidencePower,
			fullAccumulate: full, textureCount: 1, inputType: INPUT[this.options.inputType] ?? INPUT.diffuse, logTransform: !!this.options.logTransform,
			reprojectSpecular: [0, 0], historyLinear: true
		}, this.inputPlane, this.velocityPlane, this.framebufferTexture, null, this.renderTarget, null)
		this.keepData = 1
		this.prev = cam
	}
	dispose() { for (const k of ["renderTarget", "framebufferTexture", "inputPlane", "velocityPlane"]) if (this[k]) { rfx.planeFree(this.ctx, this[k]); this[k] = null } }
}

export class TRAAEffect {
	// new TRAAEffect(scene, camera, velocityDepthNormalPass, options) — src/traa/TRAAEffect.js:10-76
	constructor(scene, camera, velocityDepthNormalPass, options = defaultTemporalReprojectPassOptions) {
		this._scene = scene; this._camera = camera; this.velocityDepthNormalPass = velocityDepthNormalPass
		this.options = { ...defaultTemporalReprojectPassOptions, ...options,
			maxBlend: 0.9, neighborhoodClamp: true, neighborhoodClampIntensity: 1, neighborhoodClampRadius: 1, logTransform: true, confidencePower: 4 }   // :21-31
		this.setSize(options.width, options.height)
	}
	setSize(width, height) { this.temporalReprojectPass?.setSize(width, height) }
	reset() { this.temporalReprojectPass.reset() }
	update(renderer, inputBuffer) {
		if (!this.temporalReprojectPass) {
			this.temporalReprojectPass = new TemporalReprojectPass(this._scene, this._camera, this.velocityDepthNormalPass, inputBuffer, 1, this.options)
			this.temporalReprojectPass.setSize(inputBuffer.width, inputBuffer.height)
			this.outputPlane = rfx.planeAlloc(context(), FMT.RGBA16F, inputBuffer.width, inputBuffer.height)
			this.outputHost = new Uint16Array(4 * inputBuffer.width * inputBuffer.height)
		}
		const trp = this.temporalReprojectPass
		trp.inputTexture = inputBuffer
		trp.unjitter()                                                        // :67-72
		this.unjitteredProjectionMatrix = this._camera.projectionMatrix.clone()
		this._camera.projectionMatrix.copy(this.unjitteredProjectionMatrix)
		trp.jitter()
		trp.render(renderer)
		rfx.traaCompose(trp.ctx, trp.texture, this.outputPlane)               // traa_compose.frag:3-6
		rfx.planeDownload(trp.ctx, this.outputPlane, this.outputHost)
	}
	get outputTexture() { return this.outputHost }
	dispose() { this.temporalReprojectPass?.dispose(); if (this.outputPlane) rfx.planeFree(context(), this.outputPlane) }
}
TRAAEffect.DefaultOptions = defaultTemporalReprojectPassOptions

// -------------------------------------------------------------------------------------------------------------------------
// src/denoise/pass/PoissonDenoisePass.js:16-24
export const defaultPoissonBlurOptions = { iterations: 1, radius: 3, phi: 0.5, lumaPhi: 5, depthPhi: 2, normalPhi: 3.25, inputType: "diffuseSpecular" }

export class PoissonDenoisePass {
	// new PoissonDenoisePass(camera, textures, options) — src/denoise/pass/PoissonDenoisePass.js:26-150 (device planes in, device planes out)
	constructor(camera, textures, options = defaultPoissonBlurOptions) {
		this._camera = camera
		this.textures = Array.isArray(textures) ? textures : [textures]
		this.options = { ...defaultPoissonBlurOptions, roughnessPhi: 0, specularPhi: 0, ...options }
		this.ctx = context(); this.iterations = this.options.iterations; this.index = new BlueNoiseIndex(options.blueNoiseStart)
		reactive(this, { radius: this.options.radius, phi: this.options.phi, lumaPhi: this.options.lumaPhi, depthPhi: this.options.depthPhi,
			normalPhi: this.options.normalPhi, roughnessPhi: this.options.roughnessPhi, specularPhi: this.options.specularPhi }, () => {})
	}
	setGBufferPass(pass) { this.gbufferPlane = pass.texture; this.depthPlane = pass.depthTexture ?? this.depthPlane; this.gbufferTexture = !!pass.isGBufferPass }
	setSize(width, height) {
		this.dispose()
		const n = this.textures.length
		this.renderTargetA = Array.from({ length: n }, () => rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height))
		this.renderTargetB = Array.from({ length: n }, () => rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height))
	}
	get texture() { return this.renderTargetB }
	render() {   // :135-149 — 2 * iterations ping-pong passes
		const n = this.textures.length
		for (let i = 0; i < 2 * this.iterations; i++) {
			const horizontal = i % 2 === 0
			const src = i === 0 ? this.textures : horizontal ? this.renderTargetB : this.renderTargetA
			const dst = horizontal ? this.renderTargetA : this.renderTargetB
			rfx.poissonDenoise(this.ctx, { radius: this.radius, phi: this.phi, lumaPhi: this.lumaPhi, depthPhi: this.depthPhi, normalPhi: this.normalPhi,
				roughnessPhi: this.roughnessPhi, specularPhi: this.specularPhi, textureCount: n, isTextureSpecular: [n === 2 ? 0 : 0, n === 2 ? 1 : 0],
				gbufferTexture: this.gbufferTexture, inputLinear: i > 0 || !!this.options.inputLinear, blueNoiseIndex: this.index.value },
			this.depthPlane, this.gbufferPlane, src[0], src[1] ?? null, dst[0], dst[1] ?? null)
		}
	}
	dispose() { for (const t of [...(this.renderTargetA ?? []), ...(this.renderTargetB ?? [])]) rfx.planeFree(this.ctx, t); this.renderTargetA = this.renderTargetB = null }
}
PoissonDenoisePass.DefaultOptions = defaultPoissonBlurOptions

// -------------------------------------------------------------------------------------------------------------------------
// src/ao/AOEffect.js:8-21
export const defaultAOOptions = { resolutionScale: 1, spp: 8, distance: 2, distancePower: 1, power: 2, bias: 40, thickness: 0.075, color: [0, 0, 0],
	useNormalPass: false, velocityDepthNormalPass: null, normalTexture: null, ...defaultPoissonBlurOptions }

export class HBAOEffect {
	// new HBAOEffect(composer, camera, scene, options) — src/hbao/HBAOEffect.js:5-20 + src/ao/AOEffect.js:23-178
	// resolutionScale (0, 1]: the AO pass renders to trunc(width * scale) x trunc(height * scale) with the unrounded product as `resolution`,
	// the denoiser stays at full size (AOEffect.setSize :126-146).  normalTexture (an RGBA8 render target of view-space normals, NormalPass
	// layout) or useNormalPass (the host's NormalPass target, scene.normalRenderTarget) replaces the depth-rebuilt normal; chosen here, like
	// the reference (:48-55).
	constructor(composer, camera, scene, options = defaultAOOptions) {
		this.composer = composer; this._camera = camera; this._scene = scene
		const opts = { ...defaultAOOptions, ...options }
		checkAoScale(opts.resolutionScale)
		this._options = opts
		this.ctx = context(); this.index = new BlueNoiseIndex(options.blueNoiseStart)
		this.velocityDepthNormalPass = opts.velocityDepthNormalPass
		this.normalTarget = opts.normalTexture ?? (opts.useNormalPass ? scene?.normalRenderTarget : null)
		if (opts.useNormalPass && !this.normalTarget) throw new Error("HBAOEffect: useNormalPass needs the host's NormalPass target as scene.normalRenderTarget")
		this.lastSize = { width: 0, height: 0, resolutionScale: 0 }
		reactive(this, opts, key => { if (key === "resolutionScale") { checkAoScale(opts.resolutionScale); this.setSize(this.lastSize.width, this.lastSize.height) } })
		this.setSize(options.width ?? composer?.inputBuffer?.width, options.height ?? composer?.inputBuffer?.height)
	}
	setSize(width, height) {
		if (width === undefined || height === undefined) return
		const s = this.resolutionScale
		if (width === this.lastSize.width && height === this.lastSize.height && s === this.lastSize.resolutionScale) return
		this.dispose()
		this.width = width; this.height = height
		this.aoWidth = Math.trunc(width * s); this.aoHeight = Math.trunc(height * s)
		this.resolution = [width * s, height * s]   // AOPass.js:79-83: renderTarget.width / height as three stores them
		this.aoPlane = rfx.planeAlloc(this.ctx, FMT.RGBA16F, this.aoWidth, this.aoHeight)
		this.outputPlane = rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height)
		this.outputHost = new Uint16Array(4 * width * height)
		this.planeSource = new ReadbackPlaneSource(this.ctx, width, height)
		if (this.normalTarget) {
			this.normalW = this.normalTarget.width ?? width; this.normalH = this.normalTarget.height ?? height
			this.normalPlane = rfx.planeAlloc(this.ctx, FMT.RGBA8, this.normalW, this.normalH)
			this.normalHost = new Uint8Array(4 * this.normalW * this.normalH)
		}
		this.denoise = new PoissonDenoisePass(this._camera, [this.aoPlane], { ...this._options, normalPhi: 3.25, depthPhi: 2 })
		this.denoise.setSize(width, height)
		this.lastSize = { width, height, resolutionScale: s }
	}
	// AOEffect.js:148-154: with no denoise iteration the compose reads the AO target itself
	get texture() { return this._options.iterations > 0 ? this.denoise.texture[0] : this.aoPlane }
	initialize() {}
	// update(renderer, inputBuffer, deltaTime) — src/ao/AOEffect.js:126-178 + src/ao/AOPass.js:85-110
	update(renderer, inputBuffer) {
		const cam = cameraBlock(this._camera)
		const pv = this._camera.projectionMatrix.clone().multiply(this._camera.matrixWorldInverse)
		const planes = this.planeSource.read(renderer, { depth: this.composer.depthRenderTarget, velocity: this.velocityDepthNormalPass?.renderTarget, directLight: inputBuffer })
		if (this.normalPlane) {
			renderer.readRenderTargetPixels(this.normalTarget, 0, 0, this.normalW, this.normalH, this.normalHost)
			rfx.planeUpload(this.ctx, this.normalPlane, this.normalHost)
		}
		rfx.hbao(this.ctx, { projectionView: f32(pv), projectionInverse: cam.projectionInverse, matrixWorld: cam.matrixWorld, viewMatrix: f32(this._camera.matrixWorldInverse),
			resolution: this.resolution, aoDistance: this.distance, distancePower: this.distancePower, bias: this.bias, thickness: this.thickness, spp: this.spp,
			blueNoiseIndex: this.index.value }, planes.depth, this.aoPlane, this.normalPlane ?? null)
		this.denoise.depthPlane = planes.depth; this.denoise.gbufferPlane = planes.velocity; this.denoise.gbufferTexture = false
		this.denoise.options.inputLinear = true
		this.denoise.iterations = this._options.iterations
		this.denoise.render()
		rfx.aoCompose(this.ctx, { power: this.power, color: this.color }, planes.depth, this.texture, planes.directLight, this.outputPlane)   // ao_compose.frag:6-16
		rfx.planeDownload(this.ctx, this.outputPlane, this.outputHost)
	}
	get outputTexture() { return this.outputHost }
	dispose() {
		for (const k of ["aoPlane", "outputPlane", "normalPlane"]) if (this[k]) { rfx.planeFree(this.ctx, this[k]); this[k] = null }
		this.planeSource?.dispose(); this.denoise?.dispose()
	}
}
function checkAoScale(s) {
	if (!(typeof s === "number" && s > 0 && s <= 1)) throw new RangeError(`HBAOEffect: resolutionScale must lie in (0, 1], got ${s}`)
}
HBAOEffect.DefaultOptions = defaultAOOptions

// -------------------------------------------------------------------------------------------------------------------------
// HorizonAOEffect: an extension (the reference has no horizon march, SURVEY.md D1).  AOEffect's keys that still mean something, plus
// the march's own; spp, distancePower, bias and thickness are hbao.frag's and are not carried.
export const defaultHorizonAOOptions = { resolutionScale: 1, distance: 2, power: 2, color: [0, 0, 0], useNormalPass: false, velocityDepthNormalPass: null,
	normalTexture: null, directions: 8, steps: 32, angleBias: 0.1, intensity: 1, maxRadiusPixels: 64, ...defaultPoissonBlurOptions
}

const horizonRanges = {
	directions: [v => Number.isInteger(v) && v >= 1 && v <= 32, "an integer in 1..32"],
	steps: [v => Number.isInteger(v) && v >= 1 && v <= 64, "an integer in 1..64"],
	distance: [v => Number.isFinite(v) && v > 0, "> 0"],
	angleBias: [v => v >= 0 && v < 1, "in [0, 1)"],
	intensity: [v => Number.isFinite(v) && v >= 0, ">= 0"],
	maxRadiusPixels: [v => v >= 1, ">= 1"]
}
function checkHorizonOptions(o) {
	checkAoScale(o.resolutionScale)
	for (const [k, [ok, what]] of Object.entries(horizonRanges))
		if (typeof o[k] !== "number" || !ok(o[k])) throw new RangeError(`HorizonAOEffect: ${k} must be ${what}, got ${o[k]}`)
}

export class HorizonAOEffect extends HBAOEffect {
	// new HorizonAOEffect(composer, camera, scene, options): HBAOEffect with K6h, the horizon march (directions x steps depth taps per
	// pixel), in place of hbao.frag; target sizing, normal plane, denoise and compose are HBAOEffect's.  Options are range-checked before
	// any launch.
	constructor(composer, camera, scene, options = defaultHorizonAOOptions) {
		const opts = { ...defaultHorizonAOOptions, ...options }
		checkHorizonOptions(opts)
		super(composer, camera, scene, opts)
		for (const k of ["spp", "distancePower", "bias", "thickness"]) if (!(k in opts)) delete this._options[k]
	}
	update(renderer, inputBuffer) {
		checkHorizonOptions(this._options)
		const cam = cameraBlock(this._camera)
		const planes = this.planeSource.read(renderer, { depth: this.composer.depthRenderTarget, velocity: this.velocityDepthNormalPass?.renderTarget, directLight: inputBuffer })
		if (this.normalPlane) {
			renderer.readRenderTargetPixels(this.normalTarget, 0, 0, this.normalW, this.normalH, this.normalHost)
			rfx.planeUpload(this.ctx, this.normalPlane, this.normalHost)
		}
		rfx.hbaoHorizon(this.ctx, { projection: f32(this._camera.projectionMatrix), projectionInverse: cam.projectionInverse, matrixWorld: cam.matrixWorld,
			viewMatrix: f32(this._camera.matrixWorldInverse), resolution: this.resolution, distance: this.distance, angleBias: this.angleBias,
			intensity: this.intensity, maxRadiusPixels: this.maxRadiusPixels, directions: this.directions, steps: this.steps,
			blueNoiseIndex: this.index.value }, planes.depth, this.aoPlane, this.normalPlane ?? null)
		this.denoise.depthPlane = planes.depth; this.denoise.gbufferPlane = planes.velocity; this.denoise.gbufferTexture = false
		this.denoise.options.inputLinear = true
		this.denoise.iterations = this._options.iterations
		this.denoise.render()
		rfx.aoCompose(this.ctx, { power: this.power, color: this.color }, planes.depth, this.texture, planes.directLight, this.outputPlane)   // ao_compose.frag:6-16
		rfx.planeDownload(this.ctx, this.outputPlane, this.outputHost)
	}
}
HorizonAOEffect.DefaultOptions = defaultHorizonAOOptions

// -------------------------------------------------------------------------------------------------------------------------
export class MotionBlurEffect {
	// new MotionBlurEffect(velocityPass, options) — src/motion-blur/MotionBlurEffect.js:16-102
	constructor(velocityPass, options = { intensity: 1, jitter: 1, samples: 16 }) {
		this.velocityPass = velocityPass
		const opts = { intensity: 1, jitter: 1, samples: 16, ...options }
		this.ctx = context()
		reactive(this, opts, () => {})
	}
	initialize() {}
	setSize(width, height) {
		this.dispose()
		this.width = width; this.height = height
		this.planes = { velocity: rfx.planeAlloc(this.ctx, FMT.RGBA32F, width, height), input: rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height),
			output: rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height) }
		this.hostVel = new Float32Array(4 * width * height); this.hostIn = new Uint16Array(4 * width * height); this.outputHost = new Uint16Array(4 * width * height)
	}
	// update(renderer, inputBuffer, deltaTime) — :87-102 (frame = renderer.info.render.frame % 4096, resolution = the WINDOW size)
	update(renderer, inputBuffer, deltaTime) {
		if (!this.planes || inputBuffer.width !== this.width) this.setSize(inputBuffer.width, inputBuffer.height)
		renderer.readRenderTargetPixels(this.velocityPass.renderTarget, 0, 0, this.width, this.height, this.hostVel)
		renderer.readRenderTargetPixels(inputBuffer, 0, 0, this.width, this.height, this.hostIn)
		rfx.planeUpload(this.ctx, this.planes.velocity, this.hostVel); rfx.planeUpload(this.ctx, this.planes.input, this.hostIn)
		rfx.motionBlur(this.ctx, { intensity: this.intensity, jitter: this.jitter, deltaTime: Math.max(1 / 1000, deltaTime), samples: this.samples,
			frame: renderer.info.render.frame % 4096, resolution: [globalThis.innerWidth ?? this.width, globalThis.innerHeight ?? this.height] },
		this.planes.velocity, this.planes.input, this.planes.output)
		rfx.planeDownload(this.ctx, this.planes.output, this.outputHost)
	}
	get outputTexture() { return this.outputHost }
	dispose() { if (this.planes) for (const p of Object.values(this.planes)) rfx.planeFree(this.ctx, p); this.planes = null }
}

// ---- cosmetic effects (src/index.js:25-31) -----------------------------------------------------------------------------------------
// In the reference they are postprocessing Effects that an EffectPass merges into one fullscreen shader; here `RfxEffectPass` merges them
// into ONE launch of rfx_effects_launch (every effect samples the pass's input buffer; the colour flows from effect to effect in order).
const FX = { SHARPNESS: 1, LENS_DISTORTION: 2, GRADUAL_BACKGROUND: 3, SPARKLE: 4 }

export class SharpnessEffect {
	// new SharpnessEffect(options) — src/sharpness/SharpnessEffect.js:36-59
	constructor(options = { sharpness: 1 }) { this.fxId = FX.SHARPNESS; this.sharpness = { sharpness: 1, ...options }.sharpness }
	setSharpness(sharpness) { this.sharpness = sharpness }
	update(renderer, inputBuffer) {}
	fill(p) { p.sharpness = this.sharpness }
}

export class LensDistortionEffect {
	// new LensDistortionEffect({ alphax, alphay, aberration }) — src/lens-distortion/LensDistortionEffect.js:48-77
	constructor({ alphax = -0.05, alphay = -0.05, aberration = 1 } = {}) { this.fxId = FX.LENS_DISTORTION; Object.assign(this, { alphax, alphay, aberration }) }
	setAlphaX(value) { this.alphax = value }
	setAlphaY(value) { this.alphay = value }
	update(renderer, inputBuffer) {}
	fill(p) { Object.assign(p, { alphax: this.alphax, alphay: this.alphay, aberration: this.aberration }) }
}

export class GradualBackgroundEffect {
	// new GradualBackgroundEffect(camera, depthTexture, backgroundColor, maxDistance = 5) — src/gradual-background/GradualBackgroundEffect.js:48-70
	constructor(camera, depthTexture, backgroundColor, maxDistance = 5) { this.fxId = FX.GRADUAL_BACKGROUND; Object.assign(this, { camera, depthTexture, backgroundColor, maxDistance }) }
	setBackgroundColor(color) { this.backgroundColor = color }
	setMaxDistance(distance) { this.maxDistance = distance }
	update() {}
	fill(p) { const c = this.backgroundColor; p.backgroundColor = c.isColor ? [c.r, c.g, c.b] : c; p.maxDistance = this.maxDistance }
}

export class SparkleEffect {
	// new SparkleEffect(camera, velocityDepthNormalPass) — src/sparkle/SparkleEffect.js:102-136 (PERSPECTIVE_CAMERA is never defined there:
	// the reference's getViewZ takes the orthographic branch; definePerspectiveCamera = true gives what a host that defines it gets)
	constructor(camera, velocityDepthNormalPass, definePerspectiveCamera = false) {
		this.fxId = FX.SPARKLE; Object.assign(this, { camera, velocityDepthNormalPass, definePerspectiveCamera, spread: 1, intensity: 1 })
	}
	setSpread(spread) { this.spread = spread }
	setIntensity(intensity) { this.intensity = intensity }
	update() {}
	fill(p) { Object.assign(p, { spread: this.spread, intensity: this.intensity, sparklePerspective: this.definePerspectiveCamera ? 1 : 0 }) }
}

export class RfxEffectPass {
	// stands in for postprocessing's `new EffectPass(camera, ...effects)` when the effects are the four above
	constructor(camera, ...effects) {
		if (effects.length < 1 || effects.length > 4) throw new RangeError("RfxEffectPass: 1..4 effects")
		this.camera = camera; this.effects = effects; this.ctx = context()
	}
	setSize(width, height) {
		this.dispose()
		this.width = width; this.height = height
		this.planes = { input: rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height), output: rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height) }
		this.hostIn = new Uint16Array(4 * width * height); this.outputHost = new Uint16Array(4 * width * height)
	}
	// render(renderer, inputBuffer, outputBuffer, deltaTime, stencilTest) — the Pass contract; planes: { depth, velocity } device planes of a PlaneSource
	render(renderer, inputBuffer, outputBuffer, deltaTime, stencilTest, planes = {}) {
		if (!this.planes || inputBuffer.width !== this.width) this.setSize(inputBuffer.width, inputBuffer.height)
		renderer.readRenderTargetPixels(inputBuffer, 0, 0, this.width, this.height, this.hostIn)
		rfx.planeUpload(this.ctx, this.planes.input, this.hostIn)
		const p = { cam: cameraBlock(this.camera), count: this.effects.length, effects: this.effects.map(e => e.fxId) }
		for (const e of this.effects) { e.update(renderer, inputBuffer, deltaTime); e.fill(p) }
		rfx.effects(this.ctx, p, this.planes.input, planes.depth ?? null, planes.velocity ?? null, this.planes.output)
		rfx.planeDownload(this.ctx, this.planes.output, this.outputHost)
	}
	dispose() { if (this.planes) for (const pl of Object.values(this.planes)) rfx.planeFree(this.ctx, pl); this.planes = null }
}

export class TAAPass {
	// new TAAPass(camera) — src/taa/TAAPass.js:18-95 (renders to the screen; the RGBA8 `canvas` plane stands in for the default framebuffer)
	constructor(camera, srgbOutput = true) {
		this.camera = camera; this.srgbOutput = srgbOutput; this.ctx = context()
		this.cameraNotMovedFrames = 0; this.frame = 0; this.needsUpdate = false; this.renderToScreen = true; this.last = null
	}
	setSize(width, height) {
		this.dispose()
		this.width = width; this.height = height
		this.planes = { input: rfx.planeAlloc(this.ctx, FMT.RGBA16F, width, height), canvas: rfx.planeAlloc(this.ctx, FMT.RGBA8, width, height),
			framebufferTexture: rfx.planeAlloc(this.ctx, FMT.RGBA8, width, height) }
		this.hostIn = new Uint16Array(4 * width * height); this.outputHost = new Uint8Array(4 * width * height)
		this.needsUpdate = true
	}
	// render(renderer, inputBuffer) — :68-94
	render(renderer, inputBuffer) {
		if (!this.planes || inputBuffer.width !== this.width) this.setSize(inputBuffer.width, inputBuffer.height)
		this.frame = (this.frame + 1) % 4096
		const e = this.camera.matrixWorld.elements
		const moved = this.needsUpdate || !this.last || e.some((v, i) => Math.abs(v - this.last[i]) > 1e-6)   // didCameraMove (src/utils/SceneUtils.js:17-27)
		this.needsUpdate = false
		if (this.cameraNotMovedFrames > 0) jitter(this.width, this.height, this.camera, this.frame, 1)
		this.cameraNotMovedFrames = moved ? 0 : (this.cameraNotMovedFrames + 1) % 4096
		this.last = Array.from(e)
		renderer.readRenderTargetPixels(inputBuffer, 0, 0, this.width, this.height, this.hostIn)
		rfx.planeUpload(this.ctx, this.planes.input, this.hostIn)
		rfx.taa(this.ctx, { cameraNotMovedFrames: this.cameraNotMovedFrames, srgbOutput: this.srgbOutput ? 1 : 0 }, this.planes.input, this.planes.framebufferTexture, this.planes.canvas)
		rfx.planeDownload(this.ctx, this.planes.canvas, this.outputHost)
		const t = this.planes.canvas; this.planes.canvas = this.planes.framebufferTexture; this.planes.framebufferTexture = t   // copyFramebufferToTexture (:93)
	}
	dispose() { if (this.planes) for (const pl of Object.values(this.planes)) rfx.planeFree(this.ctx, pl); this.planes = null }
}

// ---- one Node process, several GPUs: a row-sharded group whose members live in this process (rfx_group_create_inprocess) -------------------------
// Every member owns a context (one per device), a chain with identical options (fast_math on, resolutionScale 1) and a band of rows; halo rows are recomputed, last
// frame's history rows are read in place on the member that owns them.  The per-device planes come from the caller (one PlaneSource per device).
export class InProcessGroup {
	constructor(devices, chainOptions) {
		this.ctxs = devices.map(d => rfx.ctxCreate(d))
		this.chains = this.ctxs.map(c => rfx.chainCreate(c, chainOptions))
		this.groups = this.ctxs.map((c, r) => rfx.groupCreateInprocess(c, r, devices.length))
		rfx.groupAttachChainsInprocess(this.ctxs[0], this.groups, this.chains)
	}
	setBounds(bounds) { this.groups.forEach((g, r) => rfx.groupSetBounds(this.ctxs[r], g, bounds)) }
	// planes[r]: { depth, gbuffer, velocity, directLight } device planes on device r (full frames); all members finish before the next frame starts
	render(cam, planes, cameraPos, moved) {
		this.chains.forEach((ch, r) => rfx.chainRenderSharded(this.ctxs[r], ch, cam, planes[r].depth, planes[r].gbuffer, planes[r].velocity, planes[r].directLight, cameraPos, moved))
		this.ctxs.forEach(c => rfx.ctxSync(c))
	}
	output(r, which = 0) { return rfx.chainOutput(this.ctxs[r], this.chains[r], which) }
	dispose() { this.groups.forEach(g => rfx.groupDestroy(g)); this.chains.forEach(ch => rfx.chainDestroy(ch)); this.ctxs.forEach(c => rfx.ctxDestroy(c)) }
}
