"""The GI compose (K4) and the SSGI compose (K5) across their option space, on the CPU: the case grids that
tests/test_gpu_compose_options.py runs the CUDA kernels on, which kernel path each case reaches, and the oracle against the reference's
own shaders (tests/refpins.py) at the grids' points, so that the kernels are held to the reference there.

K4 points: 200x120, 203x117, 13x9, 17x33, 90x160 and a 3840x16 strip (where (x + .5) / W * W - .5 is several ulps away from x, so the
literal bilinear fetch of a LINEAR plane takes a little of the neighbours); inputType diffuseSpecular, diffuse, and specular with and
without a scene plane; fp16 (LINEAR) or fp32 (NEAREST, denoiseMode "full_temporal") GI planes; symmetric, R2-jittered, off-axis and
orthographic cameras; a material-edge G-buffer over the synthetic depth (roughness 0 - the lensq == 0 branch of SampleGGXVNDF -, 1/256,
0.5, 1; metalness 0, 0.37, 1; zero, dim and bright emissive whose RGBE exponent bytes span 8..254; normals facing the camera, facing away
from it, and at or near +-view-Z - the other Onb basis); GI planes with high contrast between neighbours.
The `dot(viewNormal, l) < 0` flip of constructGlobalIllumination is not reached: with the one VNDF sample K4 takes (r1 = r2 = 0.25),
reflect(-V, H) stays on the normal's side for every roughness > 0 and every view direction, and at roughness 0 on a back-facing
texel H is NaN, whose comparison does not flip.  Only fp32 rounding of a nearly tangent l could take it, so deleting the flip leaves
every output of this grid unchanged (test_the_flip_of_l_is_taken_on_no_pixel counts it in float64).
K5 points: no fog, linear fog and FogExp2 with perspective and orthographic cameras, with fog parameters that put fogFactor at 0, inside
(0, 1) and at 1 on foreground pixels; isDebug; background pixels (the LINEAR scene fetch); the same sizes."""
from __future__ import annotations

from dataclasses import dataclass, replace

import numpy as np
import torch

import chain_harness as ch
import orc
import refpins
from realism_effects_b200 import abi, synth
from test_march_options_cpu import CAMERAS, make_inputs

SIZES = {(200, 120), (203, 117), (13, 9), (17, 33), (90, 160), (3840, 16)}
INPUTS = {"diffuseSpecular": abi.INPUT_DIFFUSE_SPECULAR, "diffuse": abi.INPUT_DIFFUSE, "specular": abi.INPUT_SPECULAR,
          "specular-noscene": abi.INPUT_SPECULAR}
SENTINEL = np.float32(-1234.5)  # what K4's target holds before the call; a discarded pixel keeps it


@dataclass(frozen=True)
class K4Case:
    W: int = 200
    H: int = 120
    inputs: str = "diffuseSpecular"
    gi32: bool = False  # RGBA32F NEAREST GI planes, else RGBA16F LINEAR
    camera: str = "sym"

    def __str__(self):
        return f"{self.W}x{self.H}-{self.inputs}-{'f32' if self.gi32 else 'f16'}-{self.camera}"

    @property
    def input_type(self) -> int:
        return INPUTS[self.inputs]


K4_CASES = [
    K4Case(),
    K4Case(203, 117, "diffuse", camera="jitter"),
    K4Case(13, 9, "specular", camera="offaxis"),
    K4Case(17, 33, "specular-noscene", True, "ortho"),
    K4Case(90, 160, gi32=True, camera="offaxis"),
    K4Case(3840, 16),
    K4Case(3840, 16, "specular", True, "jitter"),
    K4Case(200, 120, "diffuse", True, "ortho"),
    K4Case(203, 117, "specular-noscene"),
    K4Case(90, 160, "specular", camera="ortho"),
    K4Case(13, 9, gi32=True, camera="jitter"),
    K4Case(17, 33, "diffuse", camera="offaxis"),
    K4Case(200, 120, "specular", camera="jitter"),
    K4Case(3840, 16, "diffuse", camera="ortho"),
    K4Case(203, 117, camera="ortho"),
]

ROUGHNESS = (0.0, 1.0 / 256.0, 0.5, 1.0)
METALNESS = (0.0, 0.37, 1.0)
NORMALS = ("toward", "away", "+z", "-z", "near-z")


def material_gbuffer(depth: np.ndarray, seed: int, max_exp: int = 126) -> np.ndarray:
    """synth.pack_gbuffer over `depth` with a material drawn per pixel: 8-bit albedo, ROUGHNESS x METALNESS, emissive zero (the -1
    encoding), dim (2^-120 .. 2^-1) or bright (2^0 .. 2^max_exp; the RGBE exponent byte is at most 254), a normal of each NORMALS kind
    (world +Z is the cameras' view axis).  Background texels hold the cleared target, as synth.render_frame's do."""
    H, W = depth.shape
    n = H * W
    rng = np.random.default_rng(seed)
    albedo = np.concatenate([rng.integers(0, 256, (n, 3)) / 255.0, np.ones((n, 1))], 1)
    rough = np.asarray(ROUGHNESS)[rng.integers(0, len(ROUGHNESS), n)]
    metal = np.asarray(METALNESS)[rng.integers(0, len(METALNESS), n)]
    kind = rng.integers(0, 3, n)  # 0 zero, 1 dim, 2 bright
    e = np.where(kind == 1, rng.integers(-120, 0, n), rng.integers(0, max_exp + 1, n))
    emissive = rng.uniform(0.5, 1.0, (n, 3)) * np.exp2(e.astype(np.float64))[:, None] * (kind != 0)[:, None]
    nk = rng.integers(0, len(NORMALS), n)
    v = rng.normal(size=(n, 3))
    v[:, 2] = np.abs(v[:, 2]) + 0.2
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    normal = np.where((nk == 1)[:, None], v * [1.0, 1.0, -1.0], v)
    normal[nk == 2] = (0.0, 0.0, 1.0)
    normal[nk == 3] = (0.0, 0.0, -1.0)
    near = nk == 4
    normal[near] = np.stack([rng.uniform(-1e-3, 1e-3, near.sum()), rng.uniform(-1e-3, 1e-3, near.sum()), np.sign(rng.uniform(-1, 1, near.sum()))], 1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))  # noqa: E731
    gb = synth.pack_gbuffer(t(albedo), t(normal), t(rough), t(metal), t(emissive)).numpy().reshape(H, W, 4)
    gb[depth == 1.0] = (0.0, 0.0, 0.0, 1.0)
    return np.ascontiguousarray(gb)


def contrast_plane(H: int, W: int, seed: int, dtype) -> np.ndarray:
    """GI / scene colours in [0, 1) or [0, 64), picked per texel: neighbours differ by up to ~64x"""
    rng = np.random.default_rng(seed)
    return (rng.uniform(0.0, 1.0, (H, W, 4)) * np.where(rng.random((H, W, 1)) < 0.5, 1.0, 64.0)).astype(dtype)


_inputs: dict = {}


def inputs(W: int, H: int, camera: str) -> ch.Inputs:
    if (W, H, camera) not in _inputs:
        _inputs[(W, H, camera)] = make_inputs(W, H, camera, frames=1)
    return _inputs[(W, H, camera)]


def k4_call(case: K4Case, seed: int = 4001):
    """(params, depth, gbuffer, diffuse GI or None, specular GI or None, target before the call, scene or None): the textures
    DenoiserComposePass binds for the inputType (DenoiserComposePass.js:23-33)"""
    inp = inputs(case.W, case.H, case.camera)
    fr = inp.frames[0]
    H, W = fr["depth"].shape
    p = ch.compose_params(abi.make_camera(fr["cam"]))
    p.input_type = case.input_type
    dt = np.float32 if case.gi32 else np.float16
    d = contrast_plane(H, W, seed + 1, dt) if case.input_type != abi.INPUT_SPECULAR else None
    s = contrast_plane(H, W, seed + 2, dt) if case.input_type != abi.INPUT_DIFFUSE else None
    scene = contrast_plane(H, W, seed + 3, np.float16) if case.inputs == "specular" else None
    return p, fr["depth"], material_gbuffer(fr["depth"], seed), d, s, np.full((H, W, 4), SENTINEL, np.float32), scene


@dataclass(frozen=True)
class K5Case:
    W: int = 200
    H: int = 120
    fog: str = "none"  # "none", "linear" or "exp2"
    camera: str = "sym"  # "sym" (perspective) or "ortho"
    near: float = 8.0
    far: float = 12.0
    density: float = 0.5
    debug: bool = False

    def __str__(self):
        if self.debug:
            return f"{self.W}x{self.H}-{self.camera}-debug"
        return f"{self.W}x{self.H}-{self.camera}-{self.fog}" + {"none": "", "linear": f"-{self.near:g}-{self.far:g}", "exp2": f"-d{self.density:g}"}[self.fog]

    def params(self, cam_u: dict) -> abi.SsgiComposeParams:
        p = abi.SsgiComposeParams()
        p.use_fog, p.fog_exp2, p.perspective, p.is_debug = int(self.fog != "none"), int(self.fog == "exp2"), int(self.camera != "ortho"), int(self.debug)
        p.fog_color[:] = [0.6, 0.7, 0.8]
        p.fog_near, p.fog_far, p.fog_density = self.near, self.far, self.density
        p.camera_near, p.camera_far = float(cam_u["near"]), float(cam_u["far"])
        return p


K5_CASES = [
    K5Case(),
    K5Case(203, 117, camera="ortho"),
    K5Case(13, 9, "linear"),
    K5Case(17, 33, "linear", "ortho"),
    K5Case(90, 160, "exp2"),
    K5Case(3840, 16, "exp2", "ortho", density=1e-3),
    K5Case(3840, 16, "linear", near=0.1, far=0.5),
    K5Case(200, 120, "exp2", "ortho", density=0.25),
    K5Case(203, 117, "exp2", density=1e-3),
    K5Case(90, 160, "linear", "ortho"),
    K5Case(203, 117, debug=True),
    K5Case(13, 9, "exp2", "ortho", debug=True),
]


def k5_call(case: K5Case, seed: int = 5001):
    """(depth, gi RGBA32F, scene RGBA16F, params)"""
    fr = inputs(case.W, case.H, case.camera).frames[0]
    H, W = fr["depth"].shape
    return fr["depth"], contrast_plane(H, W, seed, np.float32), contrast_plane(H, W, seed + 1, np.float16), case.params(fr["cam"])


def fog_factor(case: K5Case, depth: np.ndarray, cam_u: dict) -> np.ndarray:
    """fogFactor of the foreground texels, in the kernels' fp32 order (exp rounded once from double, as expcr)"""
    f32 = np.float32
    d, n, f = depth[depth != 1.0].astype(f32), f32(cam_u["near"]), f32(cam_u["far"])
    gz = (n * f) / ((f - n) * d - f) if case.camera != "ortho" else d * (n - f) - n
    v = -(gz * f32(0.4))
    if case.fog == "exp2":
        k = f32(case.density)
        return f32(1.0) - np.exp((-k * k * v * v).astype(np.float64)).astype(f32)
    t = np.clip((v - f32(case.near)) / (f32(case.far) - f32(case.near)), 0.0, 1.0).astype(f32)
    return t * t * (f32(3.0) - f32(2.0) * t)


# ---- the fast chain's own K4 (c_compose) -----------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class ChainCase:
    iterations: int  # denoiseIterations: 0 = ccompose_kernel, else fused into the last Poisson pass
    tma: bool        # RFX_K3_TMA: the LINEAR passes stage their tiles through TMA
    camera: str
    W: int = 200
    H: int = 120

    def __str__(self):
        return f"{self.W}x{self.H}-it{self.iterations}-{'tma' if self.tma else 'plain'}-{self.camera}"


# The 3840-wide strips hold c_compose's centre-texel fetch to the oracle's literal bilinear one where (x + .5) / W * W - .5 is several
# ulps away from x, on the chain's own denoised planes.
CHAIN_CASES = ([ChainCase(0, True, c) for c in ("sym", "ortho")] + [ChainCase(i, t, c) for i in (1, 2) for t in (True, False) for c in ("sym", "ortho")]
               + [ChainCase(1, True, "sym", 3840, 16), ChainCase(2, False, "ortho", 3840, 16)])
_chain_inputs: dict = {}


def chain_inputs(W: int, H: int, camera: str) -> ch.Inputs:
    """3 frames of the synthetic scene with each frame's G-buffer replaced by the material-edge one (emissive up to 2^6, so that the
    march and the denoiser stay within fp16)"""
    if (W, H, camera) not in _chain_inputs:
        inp = make_inputs(W, H, camera, frames=3)
        for t, fr in enumerate(inp.frames):
            fr["gbuffer"] = material_gbuffer(fr["depth"], 8101 + t, max_exp=6)
        _chain_inputs[(W, H, camera)] = inp
    return _chain_inputs[(W, H, camera)]


def cpoisson_blocks(W: int, H: int, radius: float = 3.0) -> tuple:
    """(box fits the staged path, {interior, border} blocks of cpoisson_kernel, {interior, border} blocks of cpoisson_tma_kernel):
    chain_render_fast's reach and box, cpoisson_tma_fits, and the two kernels' block-uniform interior tests"""
    r, w, h = np.float32(radius), np.float32(W), np.float32(H)
    rx = int(np.ceil(r * max(np.float32(1.0), w / h))) + 2
    ry = int(np.ceil(r * max(np.float32(1.0), h / w))) + 2
    box_w, box_h = (16 + 2 * rx) | 1, 16 + 2 * ry
    tile = box_w * box_h * 16
    fits = box_w * 4 <= 256 and box_h <= 256 and ((tile + 127) & ~127) + tile <= 100 * 1024
    blocks = [(bx, by) for by in range(0, H, 16) for bx in range(0, W, 16)]
    plain = {"interior" if bx - rx >= 0 and bx + 15 + rx <= W - 1 and by - ry >= 0 and by + 15 + ry <= H - 1 else "border" for bx, by in blocks}
    tma = {"interior" if bx - rx >= 0 and bx - rx + box_w - 1 <= W - 1 and by - ry >= 0 and by + 15 + ry <= H - 1 else "border" for bx, by in blocks}
    return fits, plain, tma


def chain_paths(case: ChainCase) -> set:
    """the kernels (and block forms) that run c_compose in this case.  The compose rides on the last of the 2 * denoiseIterations
    Poisson passes, i = 2 * iterations - 1 >= 1: a LINEAR pass, which chain_render_fast stages through TMA when the tiles fit."""
    if case.iterations == 0:
        return {"ccompose_kernel"}
    fits, plain, tma = cpoisson_blocks(case.W, case.H)
    if case.tma and fits:
        return {f"cpoisson_tma_kernel {b}" for b in tma}
    return {f"cpoisson_kernel {b}" for b in plain}


# ---- coverage ----------------------------------------------------------------------------------------------------------------------------
def test_the_flip_of_l_is_taken_on_no_pixel():
    """constructGlobalIllumination's `if (dot(viewNormal, l) < 0.) l = -l;` restated in float64 (test_oracle_np_restatement.np_gi_compose,
    perspective cameras, even sizes): on the K4 grid's material-edge G-buffers and on the fast-chain cases' frames, the branch is taken on no composed
    pixel although a fifth of them face away from the camera"""
    from test_oracle_np_restatement import np_gi_compose

    frames = [(inputs(c.W, c.H, c.camera).frames[0], k4_call(c)[2]) for c in K4_CASES if c.camera != "ortho" and c.W % 2 == 0 and c.H % 2 == 0]
    frames += [(fr, fr["gbuffer"]) for c in {(c.W, c.H) for c in CHAIN_CASES if c.camera == "sym"} for fr in chain_inputs(c[0], c[1], "sym").frames]
    composed = away = 0
    for fr, gb in frames:
        H, W = fr["depth"].shape
        z = np.zeros((H, W, 4), np.float32)
        flips: list = []
        np_gi_compose(fr["cam"], fr["depth"], gb, z, z, z, flips=flips)
        fg = fr["depth"] != 1.0
        composed += int(fg.sum())
        away += int((orc_normals(gb[fg][:, 1])[:, 2] < 0.0).sum())
        assert not flips[0].any(), int(flips[0].sum())
    assert composed > 100000 and away > composed // 5, (composed, away)


def test_k4_grid_reaches_every_compose_configuration():
    """gi_compose_kernel: input_type x gi_f32 x fast, the specular type with and without a scene plane; every size and camera"""
    configs = {(c.input_type, c.gi32, fast) for c in K4_CASES for fast in (False, True)}
    assert configs == {(t, g, f) for t in (abi.INPUT_DIFFUSE_SPECULAR, abi.INPUT_DIFFUSE, abi.INPUT_SPECULAR) for g in (False, True) for f in (False, True)}
    assert {c.inputs for c in K4_CASES} == set(INPUTS) and {c.gi32 for c in K4_CASES if c.input_type == abi.INPUT_SPECULAR} == {False, True}
    assert {(c.W, c.H) for c in K4_CASES} == SIZES and {c.camera for c in K4_CASES} == set(CAMERAS)
    for c in K4_CASES:
        depth = inputs(c.W, c.H, c.camera).frames[0]["depth"]
        assert 0.0 < (depth == 1.0).mean() < 1.0, str(c)  # discarded pixels next to composed ones


def test_material_gbuffer_reaches_every_material_edge():
    """on the foreground of each K4 case: every roughness and metalness, the three emissive kinds with RGBE exponent bytes from 8 to 254,
    and each normal kind"""
    f32 = np.float32
    for c in K4_CASES:
        p, depth, gb, *_ = k4_call(c)
        g = gb[depth != 1.0]
        b = g[:, 2].astype(np.float64)
        rough = np.mod(b, 257.0) / 256.0
        metal = np.floor(b / (257.0 * 257.0)) / 256.0
        assert set(np.round(rough * 256).astype(int)) == {0, 1, 128, 256}, str(c)
        assert set(np.round(metal * 256).astype(int)) == {0, 95, 256}, str(c)  # 0.37 * 256 + 0.5 -> 95
        e = g[:, 3].view(np.uint32)
        ebyte = e >> 24
        assert (e == 0).any() and (ebyte < 128).any() and (ebyte > 128).any(), str(c)
        if c.W * c.H > 1000:
            assert ebyte[e != 0].min() <= 12 and ebyte.max() >= 250, (str(c), ebyte[e != 0].min(), ebyte.max())
        n = orc_normals(g[:, 1])
        assert (n[:, 2] == 1.0).any() and (n[:, 2] == -1.0).any() and (n[:, 2] < -0.2).any() and (n[:, 2] > 0.2).any(), str(c)
        assert ((np.abs(n[:, 2]) < 1.0) & (np.abs(n[:, 2]) > f32(0.9999))).any() or c.W * c.H < 1000, str(c)


def orc_normals(packed: np.ndarray) -> np.ndarray:
    """unpackNormal (gbuffer_packing.glsl:52-63) in float64"""
    h = packed.astype(np.float32).view(np.uint32)
    f = np.stack([(h & 0xFFFF).astype(np.uint16).view(np.float16), (h >> 16).astype(np.uint16).view(np.float16)], 1).astype(np.float64) * 2.0 - 1.0
    n = np.stack([f[:, 0], f[:, 1], 1.0 - np.abs(f[:, 0]) - np.abs(f[:, 1])], 1)
    t = np.maximum(-n[:, 2], 0.0)
    n[:, 0] += np.where(n[:, 0] >= 0, -t, t)
    n[:, 1] += np.where(n[:, 1] >= 0, -t, t)
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def test_k5_grid_reaches_every_branch():
    """isDebug; background (LINEAR scene) and foreground; no fog, linear fog and FogExp2 with each camera kind; fogFactor at 0, inside
    (0, 1) and at 1 for each fog kind"""
    seen = set()
    factors = {"linear": set(), "exp2": set()}
    for c in K5_CASES:
        fr = inputs(c.W, c.H, c.camera).frames[0]
        assert (c.camera == "ortho") == (fr["cam"].get("perspective", True) is False)
        if c.debug:
            seen.add("debug")
            continue
        assert 0.0 < (fr["depth"] == 1.0).mean() < 1.0, str(c)
        seen.add((c.fog, c.camera))
        if c.fog != "none":
            k = fog_factor(c, fr["depth"], fr["cam"])
            factors[c.fog] |= {"0"} if (k == 0).any() else set()
            factors[c.fog] |= {"(0,1)"} if ((k > 0) & (k < 1)).any() else set()
            factors[c.fog] |= {"1"} if (k == 1).any() else set()
    assert seen == {"debug"} | {(f, cam) for f in ("none", "linear", "exp2") for cam in ("sym", "ortho")}
    assert factors == {"linear": {"0", "(0,1)", "1"}, "exp2": {"0", "(0,1)", "1"}}, factors
    assert {(c.W, c.H) for c in K5_CASES} == SIZES


def test_chain_cases_reach_every_c_compose_path():
    """ccompose_kernel, cpoisson_kernel (interior and border blocks) and cpoisson_tma_kernel (interior and border blocks)"""
    reached = set().union(*(chain_paths(c) for c in CHAIN_CASES))
    assert reached == {"ccompose_kernel", "cpoisson_kernel interior", "cpoisson_kernel border", "cpoisson_tma_kernel interior", "cpoisson_tma_kernel border"}
    for it in (1, 2):
        for tma in (True, False):
            assert {c.camera for c in CHAIN_CASES if c.iterations == it and c.tma == tma} == {"sym", "ortho"}


def test_chain_roughness_code_equals_the_gbuffer_decode():
    """c_compose and the Poisson passes read roughness from the nrdz plane's 9-bit code (cdecode_kernel: k = clamp(mod(b, 257), 0, 256),
    nrdz_roughness: max(k / 256 - 1e-4, 0)); K4 decodes gBuffer.b (gb_roughness: max(mod(b, 257) / 256 - 1e-4, 0)).  For every roughness
    code at every metalness code, as synth.pack_gbuffer encodes them (above 2^24 the sum rounds), both give the same fp32 value."""
    f32 = np.float32
    k = np.arange(257, dtype=np.float32) / f32(256.0)
    rough, metal = np.meshgrid(k, k, indexing="ij")
    b = synth.color2float(torch.from_numpy(np.stack([rough, metal, np.zeros_like(rough)], -1))).numpy().astype(f32).ravel()
    q = (b.astype(np.float64) / 257.0).astype(f32)  # __fdiv_rn
    mod = b - f32(257.0) * np.floor(q)
    gb = np.maximum(mod / f32(256.0) - f32(1e-4), f32(0.0))
    code = np.clip(mod, 0.0, 256.0).astype(np.uint32).astype(f32)
    nrdz = np.maximum(code * f32(0.00390625) - f32(1e-4), f32(0.0))
    assert gb.dtype == np.float32 and nrdz.dtype == np.float32
    assert np.array_equal(gb.view(np.uint32), nrdz.view(np.uint32)), int((gb != nrdz).sum())


# ---- the oracle against the reference's shaders --------------------------------------------------------------------------------------
PIN_SIZES = {(200, 120): (64, 40), (203, 117): (57, 33), (90, 160): (24, 40), (13, 9): (13, 9), (17, 33): (17, 33), (3840, 16): (960, 8)}


def test_oracle_equals_reference_shaders_compose_options():
    """every K4 and K5 case of the grids at a frame of 64 x 40 or smaller (the strip: 960 x 8): the oracle's outputs, bit for bit"""
    R = refpins.ref("compose_options")
    for i, c in enumerate(K4_CASES):
        s = replace(c, W=PIN_SIZES[(c.W, c.H)][0], H=PIN_SIZES[(c.W, c.H)][1])
        p, depth, gb, d, sp, prev, scene = k4_call(s, 6001 + 10 * i)
        a = orc.gi_compose(p, depth, gb, d, sp, prev, scene=scene)
        b = R.gi_compose(p, depth, gb, d, sp, prev, scene=scene)
        assert a.tobytes() == b.tobytes(), str(c)
    for i, c in enumerate(K5_CASES):
        s = replace(c, W=PIN_SIZES[(c.W, c.H)][0], H=PIN_SIZES[(c.W, c.H)][1])
        depth, gi, scene, p = k5_call(s, 7001 + 10 * i)
        a = orc.ssgi_compose(depth, gi, scene, p)
        b = R.ssgi_compose(depth, gi, scene, p)
        assert a.tobytes() == b.tobytes(), str(c)
    refpins.done(R)
