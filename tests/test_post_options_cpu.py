"""The passes after the SSGI chain across their option space, on the CPU: HBAO (K6), AO compose (K7), motion blur (K8), TRAA compose
(K9), the cosmetic effects (Sharpness, LensDistortion, GradualBackground, Sparkle merged as one EffectPass) and TAAPass.  These are the
case grids that tests/test_gpu_post_options.py runs the CUDA kernels on, float64 restatements showing which branches the grids reach,
and the oracle against the reference's own shaders (tests/refpins.py, tag `post_options`) at the grids' points.

Sizes: 200x120, 203x117, 13x9, 90x160 and a 3840x16 strip, where (x + .5) / W * W - .5 is several ulps away from x, so a pixel-centre
LINEAR fetch takes in a little of each neighbour.  Cameras: symmetric, R2-jittered, off-axis and orthographic (test_march_options_cpu).
K6: spp 1 / 8 / 16, distance 0.3 / 2 / 8, distancePower 0 / 1 / 2.5, bias 0 / 40 / 400, thickness 0.001 / 0.075 / 5; scale 1 and a
scaled target (0.5 on 201x121), each with and without a normal plane (both instantiations of hbao_kernel's GENERAL).
`totalWeight <= 0`: the sample weight theta is 0 in exact arithmetic where the blue-noise x byte is 255 (sqrt(1 - 1) = 0 and the
other two terms are orthogonal to the normal), so on those pixels only the rounding of theta decides the branch; the grid holds such
pixels (test_k6_grid_reaches_every_branch), and the GPU test holds the kernel's bytes there to the oracle's, but a float64
restatement cannot say which side fp32 takes.
K7: power 0 / 0.5 / 1 / 2 / 3.7, black and non-black colour, AO planes with exact 0 and 1, an AO plane smaller than the frame (the
denoiser's iterations = 0 path) and background pixels.
K8: samples 1 / 2 / 7 / 16 / 33, intensity 0.25 / 1 / 3, jitter 0 / 1, deltaTime clamped at 1/1000 (uvs far outside [0, 1]),
`resolution` equal to and different from the buffer, frame 0 (the tiled lookup) and frame != 0, blue noise of 128 and 96 texels, still
pixels.
Effects: each at several values, GradualBackground with its fade at 0, inside (0, 1) and at 1, Sparkle's spread / intensity /
perspective define with both camera kinds, and all 24 orders of the four effects in one pass.
TAAPass: a 256 x 256 frame holding every finite fp16 code in R, G and B, a small frame of +-inf and NaN codes, cameraNotMovedFrames
0 / 1 / 2 / 7 / 1e6 with sRGB on and off over random history."""
from __future__ import annotations

import itertools
from dataclasses import dataclass, replace

import numpy as np

import ao_harness as ao
import chain_harness as ch
import orc
import refpins
from realism_effects_b200 import abi
from test_march_options_cpu import CAMERAS, make_inputs

SIZES = {(200, 120), (203, 117), (13, 9), (90, 160), (3840, 16)}
SENTINEL = np.float16(-1234.0)  # what K6's target holds before the call; a discarded pixel keeps it
_inputs: dict = {}


def inputs(W: int, H: int, camera: str = "sym", blue: int = 128) -> ch.Inputs:
    if (W, H, camera, blue) not in _inputs:
        _inputs[(W, H, camera, blue)] = make_inputs(W, H, camera, blue=blue, frames=1)
    return _inputs[(W, H, camera, blue)]


def color_plane(H: int, W: int, seed: int, hi: float = 1.5) -> np.ndarray:
    """RGBA16F colours in [0, hi) (alpha in [0, 1)), independent per texel: neighbours differ, so every LINEAR weight shows"""
    rng = np.random.default_rng(seed)
    c = rng.uniform(0.0, hi, (H, W, 4))
    c[..., 3] = rng.uniform(0.0, 1.0, (H, W))
    return c.astype(np.float16)


# ---- K6 -------------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class K6Case:
    W: int = 200
    H: int = 120
    spp: int = 8
    distance: float = 2.0
    power: float = 1.0
    bias: float = 40.0
    thickness: float = 0.075
    camera: str = "sym"
    scale: float = 1.0
    normal: bool = False  # an RGBA8 view-space normal plane (useNormalPass)

    def __str__(self):
        s = f"{self.W}x{self.H}-spp{self.spp}-d{self.distance:g}-p{self.power:g}-b{self.bias:g}-t{self.thickness:g}-{self.camera}"
        return s + (f"-scale{self.scale:g}" if self.scale != 1.0 else "") + ("-normal" if self.normal else "")

    @property
    def general(self) -> bool:
        return self.scale != 1.0 or self.normal


K6_CASES = [
    K6Case(),
    K6Case(203, 117, spp=1, distance=0.3, power=0.0, bias=0.0, thickness=0.001, camera="jitter"),
    K6Case(13, 9, spp=16, distance=8.0, power=2.5, bias=400.0, thickness=5.0, camera="offaxis"),
    K6Case(90, 160, distance=8.0, power=0.0, thickness=0.001, camera="ortho"),
    K6Case(3840, 16, spp=1, power=2.5, bias=0.0, thickness=5.0),
    K6Case(200, 120, spp=16, distance=0.3, bias=400.0, camera="ortho"),
    K6Case(203, 117, power=2.5, thickness=5.0, camera="offaxis"),
    K6Case(90, 160, spp=1, distance=8.0, bias=400.0, camera="jitter"),
    K6Case(3840, 16, spp=16, distance=0.3, power=0.0, thickness=0.001, camera="ortho"),
    K6Case(200, 120, normal=True),
    K6Case(203, 117, spp=16, distance=8.0, power=0.0, bias=400.0, camera="jitter", normal=True),
    K6Case(201, 121, scale=0.5),
    K6Case(201, 121, spp=1, distance=8.0, power=2.5, bias=0.0, thickness=0.001, scale=0.5, normal=True),
]


def k6_call(case: K6Case, index: int = 4711):
    """(params, depth, normal plane or None, (target W, H), resolution, target before the call)"""
    fr = inputs(case.W, case.H, case.camera).frames[0]
    (tw, th), res = ao.ao_target_size(case.W, case.H, case.scale)
    p = ao.hbao_params(fr["cam"], index, case.spp)
    p.ao_distance, p.distance_power, p.bias, p.thickness = case.distance, case.power, case.bias, case.thickness
    if case.scale != 1.0:
        p.resolution[:] = list(res)
    normal = ao.view_normal_plane(case.W, case.H, 0, fr["cam"]) if case.normal else None
    return p, fr["depth"], normal, (tw, th), res, np.full((th, tw, 4), SENTINEL, np.float16)


def k6_oracle(case: K6Case, m=None, index: int = 4711):
    """the oracle's K6: tests/orc.py's pass at scale 1 without a normal plane, tests/ao_harness.py's otherwise; `m`: a refpins
    recorder to run it through"""
    p, depth, normal, size, res, prev = k6_call(case, index)
    blue = inputs(case.W, case.H, case.camera).blue
    if not case.general:
        return (m or orc).hbao(p, depth, blue, prev)
    run = lambda impl: impl.hbao(p, depth, blue, prev, out_size=size, normal=normal, resolution=res)  # noqa: E731
    return m.arrays(lambda: run(ao.oracle), lambda: run(ao._reference())) if m else run(ao.oracle)


# ---- K7 -------------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class K7Case:
    W: int = 200
    H: int = 120
    power: float = 2.0
    color: tuple = (0.0, 0.0, 0.0)
    small: bool = False  # the AO plane is (W // 2 + 1, H // 2): the scaled AO target read directly (iterations = 0)
    camera: str = "sym"

    def __str__(self):
        return f"{self.W}x{self.H}-p{self.power:g}-c{'-'.join(f'{c:g}' for c in self.color)}" + ("-small" if self.small else "") + f"-{self.camera}"


K7_CASES = [
    K7Case(),
    K7Case(203, 117, 0.0, (0.3, 0.1, 0.9)),
    K7Case(13, 9, 0.5, camera="ortho"),
    K7Case(90, 160, 1.0, (1.0, 0.5, 0.0), camera="offaxis"),
    K7Case(3840, 16, 3.7, (0.2, 0.2, 0.2)),
    K7Case(200, 120, 2.0, (0.25, 0.5, 0.75), small=True),
    K7Case(203, 117, 3.7, small=True, camera="jitter"),
    K7Case(90, 160, 0.5, (0.1, 0.2, 0.3), camera="ortho"),
    K7Case(3840, 16, 0.0, small=True),
    K7Case(13, 9, 1.0, (0.9, 0.0, 0.4), small=True),
]


def k7_call(case: K7Case, seed: int = 7001):
    """(params, depth, AO plane, input colour): the AO plane's w channel holds exact 0 and 1 on a quarter of its texels each"""
    fr = inputs(case.W, case.H, case.camera).frames[0]
    H, W = fr["depth"].shape
    aw, ah = (W // 2 + 1, max(H // 2, 1)) if case.small else (W, H)
    rng = np.random.default_rng(seed)
    a = rng.uniform(0.0, 1.0, (ah, aw, 4))
    k = rng.integers(0, 4, (ah, aw))
    a[..., 3] = np.where(k == 0, 0.0, np.where(k == 1, 1.0, a[..., 3]))
    return ch.ao_compose_params(case.power, case.color), fr["depth"], a.astype(np.float16), color_plane(H, W, seed + 1)


def k7_oracle(case: K7Case, m=None, seed: int = 7001):
    p, depth, a, inp = k7_call(case, seed)
    if not case.small:
        return (m or orc).ao_compose(p, depth, a, inp)
    run = lambda impl: impl.ao_compose(p, depth, a, inp)  # noqa: E731
    return m.arrays(lambda: run(ao.oracle), lambda: run(ao._reference())) if m else run(ao.oracle)


# ---- K8 -------------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class K8Case:
    W: int = 200
    H: int = 120
    samples: int = 16
    intensity: float = 1.0
    jitter: float = 1.0
    dt: float = 1 / 60
    resolution: tuple | None = None  # the window size, when it differs from the buffer's
    frame: int = 7
    blue: int = 128
    vmax: float = 0.05

    def __str__(self):
        s = f"{self.W}x{self.H}-n{self.samples}-i{self.intensity:g}-j{self.jitter:g}-dt{self.dt:.4g}-f{self.frame}-blue{self.blue}-v{self.vmax:g}"
        return s + (f"-res{self.resolution[0]:g}x{self.resolution[1]:g}" if self.resolution else "")


K8_CASES = [
    K8Case(),
    K8Case(203, 117, samples=1, intensity=0.25, jitter=0.0, frame=0),
    K8Case(13, 9, samples=2, intensity=3.0, dt=1e-4, blue=96),
    K8Case(90, 160, samples=7, jitter=0.0, resolution=(333.0, 200.0), frame=0, blue=96),
    K8Case(3840, 16, samples=33, intensity=0.25, frame=3),
    K8Case(200, 120, samples=33, intensity=3.0, dt=1e-4, resolution=(150.5, 90.25), vmax=0.2),
    K8Case(203, 117, samples=16, jitter=0.0, dt=1e-4, frame=0, blue=96, vmax=0.2),
    K8Case(90, 160, samples=2, intensity=0.25, resolution=(45.0, 80.0), frame=11),
    K8Case(3840, 16, samples=7, intensity=3.0, dt=1e-4, frame=0, blue=96),
    K8Case(13, 9, samples=1, jitter=0.0, resolution=(26.0, 18.0)),
]


def k8_call(case: K8Case, seed: int = 8001):
    """(params, velocity, input colour, blue noise): the rigid-rotation velocity field with its still 8 x 8 corner"""
    inp = inputs(case.W, case.H, "sym", case.blue)
    fr = inp.frames[0]
    H, W = fr["depth"].shape
    p = ch.motion_blur_params(W, H, frame=case.frame, samples=case.samples, delta_time=case.dt, resolution=case.resolution)
    p.intensity, p.jitter = case.intensity, case.jitter
    return p, ch.rotation_velocity_field(W, H, fr["depth"], case.vmax), color_plane(H, W, seed), inp.blue


# ---- K9 -------------------------------------------------------------------------------------------------------------------------------
K9_SIZES = sorted(SIZES)


def k9_call(W: int, H: int, seed: int = 9001):
    return color_plane(H, W, seed, 64.0)


# ---- cosmetic effects -----------------------------------------------------------------------------------------------------------------
SH, LD, GB, SP = abi.FX_SHARPNESS, abi.FX_LENS_DISTORTION, abi.FX_GRADUAL_BACKGROUND, abi.FX_SPARKLE
FX_NAMES = {SH: "sharp", LD: "lens", GB: "grad", SP: "sparkle"}


@dataclass(frozen=True)
class FxCase:
    effects: tuple
    W: int = 200
    H: int = 120
    camera: str = "sym"
    sharpness: float = 1.5
    alpha: float = -0.05
    aberration: float = 1.0
    fade: str = "mid"  # where maxDistance puts GradualBackground's fade: "mid" (0, inside and 1 on one frame) or "0" / "1" everywhere
    spread: float = 1.0
    intensity: float = 1.0
    sparkle_perspective: bool = True

    def __str__(self):
        s = f"{self.W}x{self.H}-{'+'.join(FX_NAMES[e] for e in self.effects)}-{self.camera}"
        for e, t in ((SH, f"-s{self.sharpness:g}"), (LD, f"-a{self.alpha:g}-ab{self.aberration:g}"), (GB, f"-fade{self.fade}"),
                     (SP, f"-sp{self.spread:g}-i{self.intensity:g}-{'persp' if self.sparkle_perspective else 'ortho'}")):
            s += t if e in self.effects else ""
        return s


FX_CASES = [
    FxCase((SH,), sharpness=0.0),
    FxCase((SH,), 203, 117, sharpness=1.5, camera="jitter"),
    FxCase((SH,), 3840, 16, sharpness=8.0),
    FxCase((LD,), alpha=-0.3, aberration=0.0),
    FxCase((LD,), 90, 160, alpha=-0.05, aberration=1.0, camera="offaxis"),
    FxCase((LD,), 13, 9, alpha=0.2, aberration=5.0),
    FxCase((LD,), 3840, 16, alpha=0.2, aberration=5.0),
    FxCase((GB,)),
    FxCase((GB,), 203, 117, camera="ortho"),
    FxCase((GB,), 90, 160, fade="0", camera="offaxis"),
    FxCase((GB,), 13, 9, fade="1"),
    FxCase((SP,)),
    FxCase((SP,), spread=0.2, intensity=10.0),
    FxCase((SP,), 203, 117, spread=3.0, intensity=0.0, camera="jitter"),
    FxCase((SP,), 90, 160, spread=0.2, sparkle_perspective=False, camera="ortho"),
    FxCase((SP,), 200, 120, spread=1.0, intensity=10.0, sparkle_perspective=False),
    FxCase((SP,), 3840, 16, spread=0.2, intensity=10.0, camera="ortho"),
    FxCase((SH, GB, SP), 203, 117, sharpness=8.0),
] + [FxCase(order, 13, 9, sharpness=8.0, alpha=0.2, aberration=5.0, spread=0.2, intensity=10.0) for order in itertools.permutations((SH, LD, GB, SP))]


def fade_arg(cam_u: dict, depth: np.ndarray, perspective: bool) -> np.ndarray:
    """pow(distToCenter, 0.1) * 15 of GradualBackgroundEffect.js:31-46 in float64, per pixel"""
    wp = world_position(cam_u, depth, perspective)
    return (np.hypot(wp[..., 0], wp[..., 2]) + np.maximum(0.0, -wp[..., 1])) ** 0.1 * 15.0


def world_position(cam_u: dict, depth: np.ndarray, perspective: bool) -> np.ndarray:
    """getViewPosition (GradualBackgroundEffect.js:22-29, SparkleEffect.js:29-36) at the pixel centres, taken to world space, in float64"""
    H, W = depth.shape
    P = np.asarray(cam_u["projection"], np.float64).reshape(4, 4).T
    Pinv = np.asarray(cam_u["projection_inverse"], np.float64).reshape(4, 4).T
    Mw = np.asarray(cam_u["camera_matrix_world"], np.float64).reshape(4, 4).T
    n, f, d = float(cam_u["near"]), float(cam_u["far"]), depth.astype(np.float64)
    z = (n * f) / ((f - n) * d - f) if perspective else d * (n - f) - n
    ys, xs = np.mgrid[0:H, 0:W]
    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    clip = np.stack([(u - 0.5) * 2.0, (v - 0.5) * 2.0, (z - 0.5) * 2.0, np.ones_like(z)], -1) * (P[3, 2] * z + P[3, 3])[..., None]
    vp = clip @ Pinv.T
    vp[..., 2], vp[..., 3] = z, 1.0
    return (vp @ Mw.T)[..., :3]


def max_distance(case: FxCase, cam_u: dict, depth: np.ndarray) -> float:
    """maxDistance for the case's fade: "mid" puts a third of the pixels below 0, a third above 1; "0" / "1" put every pixel there"""
    a = fade_arg(cam_u, depth, bool(cam_u.get("perspective", True)))
    return {"mid": float(np.quantile(a, 0.5)) - 0.5, "0": float(a.max()) + 1.0, "1": float(a.min()) - 2.0}[case.fade]


def fx_call(case: FxCase, seed: int = 10001):
    """(params, input colour, depth, velocity): the velocity plane's depth (w) is 0 on every 7th texel, Sparkle's other early out"""
    fr = inputs(case.W, case.H, case.camera).frames[0]
    cam_u = fr["cam"]
    p = abi.make_effects_params(cam_u, case.effects, sharpness=case.sharpness, alphax=case.alpha, alphay=case.alpha, aberration=case.aberration,
                                background_color=(0.2, 0.3, 0.5), max_distance=max_distance(case, cam_u, fr["depth"]), spread=case.spread,
                                intensity=case.intensity, sparkle_perspective=case.sparkle_perspective, perspective=bool(cam_u.get("perspective", True)))
    vel = fr["velocity"].copy()
    vel.reshape(-1, 4)[::7, 3] = 0.0
    return p, color_plane(fr["depth"].shape[0], fr["depth"].shape[1], seed), fr["depth"], vel


# ---- TAAPass --------------------------------------------------------------------------------------------------------------------------
TAA_FRAMES = (0.0, 1.0, 2.0, 7.0, 1e6)


def finite_f16_codes() -> np.ndarray:
    c = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    return c[np.isfinite(c.view(np.float16))]


def taa_sweep_frame() -> np.ndarray:
    """256 x 256 RGBA16F: every finite fp16 code (negative, -0, subnormal, above 1 up to 65504) in each of R, G and B, at offsets a third
    of the codes apart; alpha in [0, 1].  W = 256: the pixel-centre LINEAR fetch returns the texel itself."""
    codes = finite_f16_codes()
    n, i = len(codes), np.arange(256 * 256)
    px = np.stack([codes[i % n], codes[(i + n // 3) % n], codes[(i + 2 * n // 3) % n],
                   (np.random.default_rng(11).uniform(0.0, 1.0, i.size)).astype(np.float16).view(np.uint16)], -1)
    return px.reshape(256, 256, 4).view(np.float16)


def taa_special_frame() -> np.ndarray:
    """24 x 10 RGBA16F: +-inf and quiet / signalling NaN codes of both signs scattered among ordinary colours (a LINEAR fetch can spread
    them into neighbours, so they stay out of the sweep)"""
    rng = np.random.default_rng(12)
    c = rng.uniform(-0.2, 1.2, (10, 24, 4)).astype(np.float16).view(np.uint16)
    special = np.array([0x7C00, 0xFC00, 0x7E00, 0xFE00, 0x7C01, 0xFD55, 0x7FFF], np.uint16)
    k = rng.integers(0, 3 * len(special), c.shape)
    c = np.where(k < len(special), special[np.minimum(k, len(special) - 1)], c)
    return c.view(np.float16)


@dataclass(frozen=True)
class TaaCase:
    frames: float
    srgb: bool
    frame: str  # "sweep" or "special"

    def __str__(self):
        return f"{self.frame}-n{self.frames:g}-{'srgb' if self.srgb else 'linear'}"

    def params(self) -> abi.TaaParams:
        p = abi.TaaParams()
        p.camera_not_moved_frames, p.srgb_output = self.frames, int(self.srgb)
        return p


TAA_CASES = [TaaCase(n, s, f) for f in ("sweep", "special") for n in TAA_FRAMES for s in (False, True)]


def taa_call(case: TaaCase):
    inp = taa_sweep_frame() if case.frame == "sweep" else taa_special_frame()
    H, W = inp.shape[:2]
    return case.params(), inp, np.random.default_rng(13 + W).integers(0, 256, (H, W, 4), dtype=np.uint8)


# ---- coverage -------------------------------------------------------------------------------------------------------------------------
def test_k6_grid_reaches_every_value_and_both_general_forms():
    assert {c.spp for c in K6_CASES} == {1, 8, 16} and {c.distance for c in K6_CASES} == {0.3, 2.0, 8.0}
    assert {c.power for c in K6_CASES} == {0.0, 1.0, 2.5} and {c.bias for c in K6_CASES} == {0.0, 40.0, 400.0}
    assert {c.thickness for c in K6_CASES} == {0.001, 0.075, 5.0} and {c.camera for c in K6_CASES} == set(CAMERAS)
    assert {(c.scale != 1.0, c.normal) for c in K6_CASES} == {(s, n) for s in (False, True) for n in (False, True)}
    assert {(c.W, c.H) for c in K6_CASES} == SIZES | {(201, 121)}
    for c in K6_CASES:
        depth = inputs(c.W, c.H, c.camera).frames[0]["depth"]
        assert 0.0 < (depth == 1.0).mean() < 1.0, str(c)  # discarded pixels next to written ones


def test_k6_grid_reaches_every_branch():
    """float64 restatement (test_oracle_np_restatement.np_hbao) of the scale-1 cases: `deltaDepth < th` taken and not taken, and
    foreground pixels whose blue-noise x byte is 255, where theta is 0 up to rounding and the rounding decides `totalWeight > 0`"""
    from test_oracle_np_restatement import np_hbao

    near, blue255 = set(), 0
    for c in K6_CASES:
        if c.general:
            continue
        p, depth, _, _, _, prev = k6_call(c)
        paths: dict = {}
        np_hbao(p, depth, inputs(c.W, c.H, c.camera).blue, prev, paths)
        near |= set(np.unique(paths["near"]).tolist())
        at = paths["blue_x"] == 255.0
        blue255 += int(at.sum())
        assert (np.abs(paths["theta"][at]) < 1e-6).all(), str(c)
        assert (paths["theta"][~at] > 1e-4).all(), str(c)
    assert near == {False, True}
    assert blue255 > 0


def test_k7_grid_reaches_every_configuration():
    assert {c.power for c in K7_CASES} == {0.0, 0.5, 1.0, 2.0, 3.7}
    assert {c.color == (0.0, 0.0, 0.0) for c in K7_CASES} == {True, False} and {c.small for c in K7_CASES} == {True, False}
    assert {(c.W, c.H) for c in K7_CASES} == SIZES
    for c in K7_CASES:
        _, depth, a, _ = k7_call(c)
        assert (a[..., 3] == 0).any() and (a[..., 3] == 1).any(), str(c)
        assert (depth > np.float32(0.9999)).any() and (depth <= np.float32(0.9999)).any(), str(c)


def test_k8_grid_reaches_every_configuration():
    """every option value; the uvs run outside [0, 1] before the clamps (startUv < 0, endUv > 1) and the still corner takes the early
    out (float64, as test_oracle_np_restatement.np_motion_blur forms them)"""
    assert {c.samples for c in K8_CASES} == {1, 2, 7, 16, 33} and {c.intensity for c in K8_CASES} == {0.25, 1.0, 3.0}
    assert {c.jitter for c in K8_CASES} == {0.0, 1.0} and {c.blue for c in K8_CASES} == {96, 128}
    assert {c.resolution is None for c in K8_CASES} == {True, False} and {c.frame == 0 for c in K8_CASES} == {True, False}
    assert {(c.W, c.H) for c in K8_CASES} == SIZES
    clamped = set()
    for c in K8_CASES:
        p, vel, _, _ = k8_call(c)
        H, W = vel.shape[:2]
        ys, xs = np.mgrid[0:H, 0:W]
        uv = np.stack([(xs + 0.5) / W, (ys + 0.5) / H], -1)
        v = vel[..., :2].astype(np.float64) * c.intensity
        speed = 0.01 / np.float64(np.float32(p.delta_time))
        lo, hi = uv - v * 0.5 * speed, uv + v * 0.5 * speed  # startUv, endUv before the clamps (jitter 0: no blue-noise offset)
        moved = (vel[..., :2].astype(np.float64) ** 2).sum(-1) > 1e-9
        assert (~moved).any() and moved.any(), str(c)
        if c.jitter == 0.0 and (lo[moved] < 0).any() and (hi[moved] > 1).any():
            clamped.add(c.dt)
        assert np.float32(p.delta_time) == np.float32(max(1 / 1000, c.dt))
    assert 1e-4 in clamped


def fx_paths(case: FxCase) -> set:
    """the branches of the case's effects, in float64: GradualBackground's fade at 0, inside (0, 1), at 1; Sparkle's early outs (depth 0
    or 1, worldPos.y < 0.01) and its sparkling pixels; LensDistortion fetches outside [0, 1]"""
    p, _, depth, vel = fx_call(case)
    fr = inputs(case.W, case.H, case.camera).frames[0]
    out = set()
    if GB in case.effects:
        f = np.clip(fade_arg(fr["cam"], depth, bool(fr["cam"].get("perspective", True))) - p.max_distance, 0.0, 1.0)
        out |= {n for n, m in (("fade 0", f == 0), ("fade (0,1)", (f > 0) & (f < 1)), ("fade 1", f == 1)) if m.any()}
    if SP in case.effects:
        d = vel[..., 3]
        out |= {"sparkle depth 0"} if (d == 0).any() else set()
        out |= {"sparkle depth 1"} if (d == 1).any() else set()
        y = world_position(fr["cam"], d, case.sparkle_perspective)[..., 1]
        fg = (d != 0) & (d != 1)
        out |= {"sparkle y < 0.01"} if (fg & (y < 0.01)).any() else set()
        out |= {"sparkle"} if (fg & (y >= 0.01)).any() else set()
    if LD in case.effects:
        H, W = depth.shape
        ys, xs = np.mgrid[0:H, 0:W]
        x, y = 2.0 * (xs + 0.5) / W - 1.0, 2.0 * (ys + 0.5) / H - 1.0
        r = x * x + y * y
        q = (x / (1.0 - case.alpha * r)) ** 2 + (y / (1.0 - case.alpha * r)) ** 2
        u, v = (x / (1.0 - case.alpha * q) + 1.0) / 2.0, (y / (1.0 - case.alpha * q) + 1.0) / 2.0
        fetch = [(u - case.aberration / W, v), (u, v - case.aberration / H), (u - case.aberration / W, v - case.aberration / H)]
        if any(((a < 0) | (a > 1) | (b < 0) | (b > 1)).any() for a, b in fetch):
            out.add("lens outside")
    return out


def test_fx_grid_reaches_every_value_and_branch():
    single = [c for c in FX_CASES if len(c.effects) == 1]
    assert {c.sharpness for c in single if c.effects == (SH,)} == {0.0, 1.5, 8.0}
    assert {c.alpha for c in single if c.effects == (LD,)} == {-0.3, -0.05, 0.2}
    assert {c.aberration for c in single if c.effects == (LD,)} == {0.0, 1.0, 5.0}
    sp = [c for c in single if c.effects == (SP,)]
    assert {c.spread for c in sp} == {0.2, 1.0, 3.0} and {c.intensity for c in sp} == {0.0, 1.0, 10.0}
    assert {(c.sparkle_perspective, c.camera == "ortho") for c in sp} == {(a, b) for a in (False, True) for b in (False, True)}
    assert {c.camera for c in FX_CASES} == set(CAMERAS) and {(c.W, c.H) for c in FX_CASES} == SIZES
    assert {c.effects for c in FX_CASES if len(c.effects) == 4} == set(itertools.permutations((SH, LD, GB, SP)))
    reached = set().union(*(fx_paths(c) for c in FX_CASES))
    assert reached == {"fade 0", "fade (0,1)", "fade 1", "sparkle depth 0", "sparkle depth 1", "sparkle y < 0.01", "sparkle", "lens outside"}, reached
    for c in FX_CASES:
        if c.effects == (GB,) and c.fade == "mid":
            assert {"fade 0", "fade (0,1)", "fade 1"} <= fx_paths(c), str(c)


def test_taa_frames_hold_every_code_and_reach_every_branch():
    """the sweep holds every finite fp16 code in each colour channel; in float64, texels whose 8-bit rounding lies inside the 2e-3 tie
    window (the exact re-evaluation runs) for every frame count up to 7 with sRGB on, and negative channels with cameraNotMovedFrames > 0"""
    sweep = taa_sweep_frame()
    codes = set(finite_f16_codes().tolist())
    for ch_ in range(3):
        assert set(sweep[..., ch_].view(np.uint16).ravel().tolist()) == codes
    sp = taa_special_frame().view(np.uint16)
    assert {0x7C00, 0xFC00} <= set(sp.ravel().tolist()) and np.isnan(sp.view(np.float16)).any()
    for c in TAA_CASES:
        if c.frame != "sweep" or not c.srgb:
            continue
        p, inp, hist = taa_call(c)
        v = inp[..., :3].astype(np.float64)
        with np.errstate(invalid="ignore"):
            a = (v <= 0.0031308).astype(np.float64)
            s = (np.power(v, 0.41666) * 1.055 - 0.055) * (1.0 - a) + v * 12.92 * a  # mix(): pow's NaN survives a = 1
        t = 1.0 / (c.frames + 1.0)
        o = s if c.frames == 0 else hist[..., :3] / 255.0 * (1.0 - t) + s * t
        q = np.clip(o, 0.0, 1.0) * 255.0
        assert (np.abs((q - np.floor(q)) - 0.5) < 2e-3).sum() > 10 or c.frames == 1e6, str(c)  # at 1e6 the history's code decides
        if c.frames > 0:
            assert (v < 0).any() and np.isnan(o[v < 0]).all(), str(c)


# ---- the oracle against the reference's shaders --------------------------------------------------------------------------------------
PIN_SIZES = {(200, 120): (64, 40), (203, 117): (57, 33), (201, 121): (67, 41), (90, 160): (24, 40), (13, 9): (13, 9), (3840, 16): (960, 8)}


def pin(case):
    return replace(case, W=PIN_SIZES[(case.W, case.H)][0], H=PIN_SIZES[(case.W, case.H)][1])


def test_oracle_equals_reference_shaders_post_options():
    """every case of the grids at a frame of 67 x 41 or smaller (the strip: 960 x 8; TAAPass at its own sizes): the oracle's outputs,
    bit for bit"""
    R = refpins.ref("post_options")
    for c in K6_CASES:
        k6_oracle(pin(c), R)
    for c in K7_CASES:
        k7_oracle(pin(c), R)
    for c in K8_CASES:
        R.motion_blur(*k8_call(pin(c)))
    for W, H in K9_SIZES:
        W, H = PIN_SIZES[(W, H)]
        R.traa_compose(k9_call(W, H))
    for c in FX_CASES:
        R.effects(*fx_call(pin(c)))
    for c in TAA_CASES:
        R.taa(*taa_call(c))
    refpins.done(R)
