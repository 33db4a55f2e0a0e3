"""Reduced-resolution AO (AOEffect's resolutionScale) and K6's normal-texture input — TEST INFRASTRUCTURE.

* `oracle`: tests/ao_oracle.cpp (the CPU oracle of oracle/rfx_oracle.cpp extended by the AO target's own size, the `resolution`
  uniform, an RGBA8 normal plane, and Poisson / compose inputs smaller than the pass), bound with ctypes and built on first use into
  build/ (git-ignored) with oracle/Makefile's flags.
* `reference`: the same calls on the reference's own shaders (tests/refglsl.py; needs the reference checkout or prebuilt libraries).
* the host values the reference's JS derives: the AO target of a scale, the NormalPass plane of a synthetic frame, K6's uniforms.
* pins: digests of what the reference's shaders computed for tests/test_reference_glsl_ao.py, in tests/golden/reference_pins_ao.json
  (minted by tests/golden/make_golden_ao.py), so the comparison runs bit for bit without the checkout.

Both `oracle` and `reference` have `hbao(p, depth, blue_noise, out_prev, *, out_size=None, normal=None, resolution=None)`,
`poisson_denoise(...)` with the signature of tests/orc.py (in0 / in1 may be smaller than depth) and `ao_compose(p, depth, ao, inp)`
(ao of any size), so chain_harness.ao_denoise(m, ...) drives either.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import subprocess
import types

import numpy as np

from realism_effects_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "ao_oracle.cpp")
SO = os.path.join(ROOT, "build", "librfx_oracle_ao.so")
PINS = os.path.join(ROOT, "tests", "golden", "reference_pins_ao.json")
_DEPS = [SRC, os.path.join(ROOT, "oracle", "rfx_oracle.cpp"), os.path.join(ROOT, "oracle", "glsl.h"), os.path.join(ROOT, "oracle", "Makefile"),
         os.path.join(ROOT, "include", "rfx.h")]
# oracle/Makefile's CXXFLAGS: the same fp32 lowering as the oracle it extends
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wall", "-Wno-unused-function",
            "-Wno-unused-variable", "-Wno-unused-but-set-variable"]


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
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f16(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16) if a.dtype == np.float16 else a


def _hbao_oracle(p: abi.HbaoParams, depth, blue_noise, out_prev, *, out_size=None, normal=None, resolution=None):
    DH, DW = depth.shape
    W, H = out_size or (DW, DH)
    rx, ry = resolution or (W, H)
    out = np.array(_f16(out_prev), copy=True)
    assert out.shape == (H, W, 4), (out.shape, (H, W))
    bn = np.ascontiguousarray(blue_noise, np.uint8)
    n = None if normal is None else np.ascontiguousarray(normal, np.uint8)
    _L().orc_ao_hbao(C.byref(p), C.c_int(W), C.c_int(H), C.c_float(rx), C.c_float(ry), _p(np.ascontiguousarray(depth, np.float32)), C.c_int(DW),
                     C.c_int(DH), _p(n), C.c_int(0 if n is None else n.shape[1]), C.c_int(0 if n is None else n.shape[0]), _p(bn), C.c_int(bn.shape[1]),
                     C.c_int(bn.shape[0]), _p(out))
    return out.view(np.float16)


def _poisson_oracle(p: abi.PoissonParams, depth, gbuffer_or_normal, in0, in1, blue_noise, out0_prev, out1_prev):
    H, W = depth.shape
    in_half = in0.dtype in (np.float16, np.uint16)
    i0 = _f16(in0) if in_half else np.ascontiguousarray(in0, np.float32)
    i1 = None if in1 is None else (_f16(in1) if in_half else np.ascontiguousarray(in1, np.float32))
    o0 = np.array(_f16(out0_prev), copy=True)
    o1 = None if out1_prev is None else np.array(_f16(out1_prev), copy=True)
    bn = np.ascontiguousarray(blue_noise, np.uint8)
    _L().orc_ao_poisson_denoise(C.byref(p), C.c_int(W), C.c_int(H), _p(np.ascontiguousarray(depth, np.float32)),
                                _p(np.ascontiguousarray(gbuffer_or_normal, np.float32)), _p(i0), _p(i1), C.c_int(int(in_half)), C.c_int(in0.shape[1]),
                                C.c_int(in0.shape[0]), _p(bn), C.c_int(bn.shape[1]), C.c_int(bn.shape[0]), _p(o0), _p(o1))
    return o0.view(np.float16), None if o1 is None else o1.view(np.float16)


def _ao_compose_oracle(p: abi.AoComposeParams, depth, ao, inp):
    H, W = depth.shape
    out = np.zeros((H, W, 4), np.uint16)
    a = _f16(ao)
    _L().orc_ao_ao_compose(C.byref(p), C.c_int(W), C.c_int(H), _p(np.ascontiguousarray(depth, np.float32)), _p(a), C.c_int(a.shape[1]), C.c_int(a.shape[0]),
                           _p(_f16(inp)), _p(out))
    return out.view(np.float16)


oracle = types.SimpleNamespace(hbao=_hbao_oracle, poisson_denoise=_poisson_oracle, ao_compose=_ao_compose_oracle)


def _hbao_reference(p: abi.HbaoParams, depth, blue_noise, out_prev, *, out_size=None, normal=None, resolution=None):
    """AOPass.render (src/ao/AOPass.js:85-110, uniforms :36-54) on the AO target of AOEffect.setSize (src/ao/AOEffect.js:126-146):
    Shader.run at the target size, `resolution` and blueNoiseRepeat from the unrounded target size (:79-83, :98-105); with a normal
    plane the useNormalTexture define (AOEffect.js:48-55), normalTexture RGBA8 NEAREST and viewMatrix = camera.matrixWorldInverse"""
    import refglsl as R

    H, W = depth.shape
    if out_size:
        W, H = out_size
    res = list(resolution or (W, H))
    s = R.Shader.get("hbao", spp=int(p.spp), **(dict(use_normal_texture=True) if normal is not None else {}))
    s.set(optional=("frame", "blueNoiseRepeat", "cameraNear", "cameraFar", "viewMatrix"), projectionViewMatrix=list(p.projection_view),
          projectionMatrixInverse=list(p.projection_inverse), cameraMatrixWorld=list(p.camera_matrix_world), aoDistance=float(p.ao_distance),
          distancePower=float(p.distance_power), bias=float(p.bias), thickness=float(p.thickness), resolution=res, frame=0,
          blueNoiseRepeat=[res[0] / 128, res[1] / 128], viewMatrix=list(p.view_matrix))
    s.tex("depthTexture", depth, R.F_R32F)
    s.tex("normalTexture", normal, R.F_RGBA8, optional=True)
    s.tex("blueNoiseTexture", blue_noise, R.F_RGBA8, repeat=True)
    s.set(blueNoiseSize=[blue_noise.shape[1], blue_noise.shape[0]], blueNoiseIndex=int(p.blue_noise_index))
    return s.run(W, H, [(R.F_RGBA16F, out_prev)])[0]


def _reference():
    """refglsl's Poisson and compose wiring takes every texture at its own size already"""
    import refglsl as R

    return types.SimpleNamespace(hbao=_hbao_reference, poisson_denoise=R.poisson_denoise, ao_compose=R.ao_compose)


# ------------------------------------------------------------------------------------------------------------------ host values
def ao_target_size(width: int, height: int, scale: float):
    """AOEffect.setSize: the AO target of resolutionScale `scale` -> ((W, H), resolution).  three's WebGLRenderTarget keeps
    width * scale unrounded (the `resolution` uniform, AOPass.js:79-83); GL truncates it for the texture."""
    return (int(width * scale), int(height * scale)), (width * scale, height * scale)


def hbao_params(cam_u: dict, index: int, spp: int = 8, resolution=None) -> abi.HbaoParams:
    """chain_harness.hbao_params plus the uniforms of the new fields: viewMatrix (AOPass.js:41) and resolution ({0, 0}: the target's size)"""
    import chain_harness as ch

    p = ch.hbao_params(cam_u, index, spp)
    abi.set_f16(p.view_matrix, cam_u["view_matrix"])
    if resolution is not None:
        p.resolution[:] = [float(resolution[0]), float(resolution[1])]
    return p


def view_normal_plane(width: int, height: int, t: int, cam_u: dict) -> np.ndarray:
    """postprocessing's NormalPass target for synthetic frame `t` (chain_harness.make_inputs' defaults): the view-space normal packed
    as rgb = n * 0.5 + 0.5 in RGBA8, from the scene's world normals rotated by the view matrix.  (H, W, 4) uint8."""
    from realism_effects_b200 import synth

    n = synth.render_frame(width, height, t).soa["normal"][..., :3].double().numpy()
    V = np.asarray(cam_u["view_matrix"], np.float64).reshape(4, 4).T
    v = n @ V[:3, :3].T
    v /= np.maximum(np.linalg.norm(v, axis=-1, keepdims=True), 1e-12)
    out = np.full((height, width, 4), 255, np.uint8)
    out[..., :3] = np.clip(np.round((v * 0.5 + 0.5) * 255.0), 0, 255).astype(np.uint8)
    return out


# ------------------------------------------------------------------------------------------------------------------ pins
def digest(a) -> str:
    """the first 64 bits of the SHA-256 of the array's bytes"""
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def check_pins(tag: str, arrays: list):
    """`arrays` (computed on the oracle) must have the digests the reference's shaders' outputs had"""
    with open(PINS, encoding="utf-8") as f:
        want = json.load(f)[tag]
    got = [digest(a) for a in arrays]
    assert len(got) == len(want), f"{tag}: {len(got)} outputs, {len(want)} recorded (re-mint tests/golden/make_golden_ao.py)"
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"{tag}: outputs {bad} differ from the reference's shaders"
