"""Debug views of SSGIEffect's `outputTexture` (src/ssgi/SSGIEffect.js:228-251) — TEST INFRASTRUCTURE.

* `oracle`: tests/debug_oracle.cpp (the CPU oracle of oracle/rfx_oracle.cpp extended by GBufferDebugPass and K5's isDebug branch on a
  view of any format and size), bound with ctypes and built on first use into build/ (git-ignored) with oracle/Makefile's flags.
* `reference`: the same calls on the reference's own shaders (tests/refglsl.py; needs the reference checkout or prebuilt libraries).
  GBufferDebugPass's shader is the template literal of src/gbuffer/debug/GBufferDebugPass.js, assembled like the other template-literal
  passes of oracle/ref/assemble.py.
* pins: digests of what the reference's shaders computed for tests/test_debug_views_cpu.py, in tests/golden/reference_pins_debug.json
  (minted by tests/golden/make_golden_debug.py), so the comparison runs bit for bit without the checkout.
* the inputs: a synthetic frame whose G-buffer has background (cleared) texels and transparent-black albedo texels, and K5 views of every
  source kind.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import re
import subprocess
import types

import numpy as np

from realism_effects_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "debug_oracle.cpp")
SO = os.path.join(ROOT, "build", "librfx_oracle_debug.so")
PINS = os.path.join(ROOT, "tests", "golden", "reference_pins_debug.json")
_DEPS = [SRC, os.path.join(ROOT, "oracle", "rfx_oracle.cpp"), os.path.join(ROOT, "oracle", "glsl.h"), os.path.join(ROOT, "oracle", "Makefile"),
         os.path.join(ROOT, "include", "rfx.h")]
# oracle/Makefile's CXXFLAGS: the same fp32 lowering as the oracle it extends
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wall", "-Wno-unused-function",
            "-Wno-unused-variable", "-Wno-unused-but-set-variable"]

# the strings SSGIEffect's setter maps to GBufferDebugPass modes (SSGIEffect.js:237-239); an unknown string gives mode -1
MODES = abi.GBUFFER_DEBUG_MODES


def build(force: bool = False) -> str:
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in _DEPS):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        tmp = SO + f".{os.getpid()}.tmp"
        subprocess.check_call(["g++", *CXXFLAGS, "-shared", "-o", tmp, SRC])
        os.replace(tmp, SO)
    return SO


_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _fmt(view: np.ndarray) -> int:
    if view.ndim == 2:
        return abi.FMT_R32F
    return abi.FMT_RGBA16F if view.dtype in (np.float16, np.uint16) else abi.FMT_RGBA32F


def _gbuffer_debug_oracle(mode: int, gbuffer):
    g = np.ascontiguousarray(gbuffer, np.float32)
    H, W = g.shape[:2]
    out = np.zeros((H, W, 4), np.float32)
    _L().orc_dbg_gbuffer_debug(C.c_int(int(mode)), C.c_int(W), C.c_int(H), _p(g), _p(out))
    return out


def _ssgi_compose_debug_oracle(view, out_size):
    """K5 with isDebug into a W x H RGBA16F target; `view`: (h, w) float32 depth, (h, w, 4) float16 (LINEAR) or float32 (NEAREST)"""
    W, H = out_size
    v = np.ascontiguousarray(view)
    if v.dtype == np.float16:
        v = v.view(np.uint16)
    out = np.zeros((H, W, 4), np.uint16)
    _L().orc_dbg_ssgi_compose_debug(C.c_int(W), C.c_int(H), C.c_int(_fmt(view)), _p(v), C.c_int(v.shape[1]), C.c_int(v.shape[0]), _p(out))
    return out.view(np.float16)


oracle = types.SimpleNamespace(gbuffer_debug=_gbuffer_debug_oracle, ssgi_compose_debug=_ssgi_compose_debug_oracle)


# ------------------------------------------------------------------------------------------------------------------ the reference
def gbuffer_debug_glsl() -> str:
    """GBufferDebugPass.js:19-57: the template literal with ${gbuffer_packing}, through WebGLProgram like every ShaderMaterial"""
    import refglsl as R

    js = R.assemble.read("gbuffer/debug/GBufferDebugPass.js")
    frag = re.search(r"fragmentShader:\s*/\*\s*glsl\s*\*/\s*`(.*?)`", js, flags=re.S).group(1)
    frag = frag.replace("${gbuffer_packing}", R.assemble.read("gbuffer/shader/gbuffer_packing.glsl"))
    return R.assemble.finish(frag, {})


_gb_shader = None


def _gbuffer_debug_reference(mode: int, gbuffer):
    """GBufferDebugPass.render with uniforms {gBufferTexture, mode} (:58-61).  `depthTexture` is declared by the shader but is not in
    that list, and three uploads only the uniforms a material lists, so the sampler keeps GL's default unit 0 — the unit of the first
    sampler three allocates, gBufferTexture.  It is therefore bound to the G-buffer plane here: depth == 0. holds where the packed albedo
    bits compare equal to zero (three's own source is not needed for this; it rests on its documented uniform-upload behaviour)."""
    import refglsl as R

    global _gb_shader
    if _gb_shader is None:
        _gb_shader = R.Shader("gbuffer_debug", glsl=gbuffer_debug_glsl())
    s = _gb_shader
    s.reset()
    g = np.ascontiguousarray(gbuffer, np.float32)
    H, W = g.shape[:2]
    s.set(mode=int(mode))
    s.tex("gBufferTexture", g, R.F_RGBA32F)
    s.tex("depthTexture", g, R.F_RGBA32F)
    return s.run(W, H, [(R.F_RGBA32F, None)])[0]


def _ssgi_compose_debug_reference(view, out_size):
    """SSGIEffect.update with isDebug (SSGIEffect.js:402): inputTexture = the view with its own sampler — FloatType targets NEAREST,
    the Poisson targets (HalfFloat) LINEAR, a depth texture (d, 0, 0, 1)"""
    import refglsl as R

    W, H = out_size
    s = R.Shader.get("ssgi_compose", fog=False, fog_exp2=False, perspective=True)
    s.set(optional=("fogColor", "fogNear", "fogFar", "fogDensity"), isDebug=1, cameraNear=0.1, cameraFar=1000.0)
    f = _fmt(view)
    s.tex("depthTexture", np.ones((H, W), np.float32), R.F_R32F)
    s.tex("inputTexture", view, {abi.FMT_R32F: R.F_R32F, abi.FMT_RGBA16F: R.F_RGBA16F, abi.FMT_RGBA32F: R.F_RGBA32F}[f], linear=f == abi.FMT_RGBA16F)
    s.tex("sceneTexture", np.zeros((H, W, 4), np.float16), R.F_RGBA16F, linear=True)
    return s.run(W, H, [(R.F_RGBA16F, None)])[0]


reference = types.SimpleNamespace(gbuffer_debug=_gbuffer_debug_reference, ssgi_compose_debug=_ssgi_compose_debug_reference)


def reference_available() -> bool:
    import refglsl as R

    return R.assemble.available()


# ------------------------------------------------------------------------------------------------------------------ inputs
def debug_frame(width: int, height: int, t: int = 0) -> dict:
    """a synthetic frame (synth.render_frame) whose G-buffer has the cleared texel (all zero) on the background and two blocks of
    transparent-black albedo: packed albedo bits 0x00000000 and 0x80000000 (-0.0, alpha byte 128), the other channels kept"""
    from realism_effects_b200 import synth

    fr = synth.render_frame(width, height, t)
    depth = fr.depth.cpu().numpy()
    gb = np.array(fr.gbuffer.cpu().numpy(), np.float32, copy=True)
    gb[depth == 1.0] = 0.0
    bits = gb.view(np.uint32)
    h4, w4 = max(height // 4, 1), max(width // 4, 1)
    bits[h4:2 * h4, w4:2 * w4, 0] = 0x00000000
    bits[2 * h4:3 * h4, 2 * w4:3 * w4, 0] = 0x80000000
    return dict(depth=depth, gbuffer=gb, velocity=fr.velocity.cpu().numpy(), direct=fr.direct_light.cpu().numpy(), cam=fr.cam.uniforms())


def rgbe_gbuffer(width: int = 64, height: int = 16) -> np.ndarray:
    """a G-buffer whose emissive texels (gBuffer.a, vec4ToFloat(encodeRGBE8(...)) bits) take every exponent byte 0..255 with varied
    mantissa bytes, so that GBufferDebugPass's emissive mode sees every fExp decodeRGBE8 can get; albedo is opaque and non-zero"""
    rng = np.random.default_rng(11)
    n = width * height
    e = np.arange(n, dtype=np.uint32) % 256
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint32)
    g = np.zeros((n, 4), np.uint32)
    g[:, 0] = 0x3F102030  # non-zero albedo: not masked by the pass's depth test
    g[:, 3] = rgb[:, 0] | (rgb[:, 1] << 8) | (rgb[:, 2] << 16) | (e << 24)
    return g.view(np.float32).reshape(height, width, 4)


def k5_views(width: int, height: int, seed: int = 7) -> list:
    """(name, view) for K5's debug branch at a width x height target: every source kind"""
    rng = np.random.default_rng(seed)
    fr = debug_frame(width, height)
    views = [("composed", rng.normal(0.5, 1.0, (height, width, 4)).astype(np.float32)),
             ("depth", fr["depth"]), ("velocity", fr["velocity"]), ("gbuffer", fr["gbuffer"]),
             ("dnB", rng.normal(0.5, 1.0, (height, width, 4)).astype(np.float16))]
    for s in (0.5, 0.75):  # the SSGI target of resolutionScale s: (int)(width * s) x (int)(height * s), fetched NEAREST by uv
        views.append((f"ssgi_scale{s}", rng.normal(0.5, 1.0, (int(height * s), int(width * s), 4)).astype(np.float32)))
    return views


# ------------------------------------------------------------------------------------------------------------------ pins
def digest(a) -> str:
    """the first 64 bits of the SHA-256 of the array's bytes"""
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def check_pins(tag: str, arrays: list):
    """`arrays` (computed on the oracle) must have the digests the reference's shaders' outputs had"""
    with open(PINS, encoding="utf-8") as f:
        want = json.load(f)[tag]
    got = [digest(a) for a in arrays]
    assert len(got) == len(want), f"{tag}: {len(got)} outputs, {len(want)} recorded (re-mint tests/golden/make_golden_debug.py)"
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"{tag}: outputs {bad} differ from the reference's shaders"


# the cases of the pins: (tag, [outputs]) for module m (oracle or reference)
GB_SIZES = [(64, 36), (61, 35)]
K5_SIZES = [(64, 36), (203, 117)]


def pin_cases(m) -> dict:
    out = {}
    for W, H in GB_SIZES:
        g = debug_frame(W, H)["gbuffer"]
        out[f"gbuffer_debug_{W}x{H}"] = [m.gbuffer_debug(mode, g) for mode in (*range(6), -1)]
    out["gbuffer_debug_rgbe"] = [m.gbuffer_debug(5, rgbe_gbuffer())]
    for W, H in K5_SIZES:
        out[f"k5_debug_{W}x{H}"] = [m.ssgi_compose_debug(v, (W, H)) for _, v in k5_views(W, H)]
    return out
