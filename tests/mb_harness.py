"""TRAAEffect + MotionBlurEffect as one EffectPass — TEST INFRASTRUCTURE.

* `oracle`: tests/mb_oracle.cpp (the CPU oracle of oracle/rfx_oracle.cpp extended by the merged pass), bound with ctypes and built on
  first use into build/ (git-ignored) with oracle/Makefile's flags.
* `reference`: the same pass on the reference's own shaders (tests/refglsl.py; needs the reference checkout or prebuilt libraries).
  postprocessing merges the effects' mainImage()s into one program and hands the first one's outputColor to the second as inputColor.
  Here traa_compose.frag runs into an RGBA32F plane, and motion_blur.frag reads that plane as its inputBuffer (NEAREST at the pixel
  centre: the fp32 colour itself) with inputTexture bound to the pass's input buffer, as MotionBlurEffect.update binds it
  (src/motion-blur/MotionBlurEffect.js:87-90).  That is the merged program's arithmetic; tests/refglsl.effects chains the cosmetic
  effects the same way.
* pins: digests of what the reference's shaders computed for tests/test_traa_motion_blur_cpu.py, in tests/golden/reference_pins_mb.json
  (minted by tests/golden/make_golden_mb.py), so the comparison runs bit for bit without the checkout.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np

from realism_effects_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "mb_oracle.cpp")
SO = os.path.join(ROOT, "build", "librfx_oracle_mb.so")
PINS = os.path.join(ROOT, "tests", "golden", "reference_pins_mb.json")
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


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f16(a) -> np.ndarray:
    a = np.ascontiguousarray(a)
    return a.view(np.uint16) if a.dtype == np.float16 else a


def oracle(p: abi.MotionBlurParams, velocity, acc, inp, blue_noise) -> np.ndarray:
    """the merged pass on the oracle: velocity RGBA32F, acc / inp RGBA16F (H, W, 4); returns RGBA16F"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    H, W = velocity.shape[:2]
    out = np.zeros((H, W, 4), np.uint16)
    vel = np.ascontiguousarray(velocity, np.float32)
    a, i, bn = _f16(acc), _f16(inp), np.ascontiguousarray(blue_noise, np.uint8)
    _lib.orc_traa_motion_blur(C.byref(p), C.c_int(W), C.c_int(H), _p(vel), _p(a), _p(i), _p(bn), C.c_int(bn.shape[1]), C.c_int(bn.shape[0]), _p(out))
    return out.view(np.float16)


def reference(p: abi.MotionBlurParams, velocity, acc, inp, blue_noise) -> np.ndarray:
    """the merged pass on the reference's shaders (see the module docstring)"""
    import refglsl as R

    H, W = velocity.shape[:2]
    s = R.Shader.get("traa_compose")  # TRAAEffect  src/traa/TRAAEffect.js:11-15,63
    s.tex("accumulatedTexture", acc, R.F_RGBA16F, linear=True)
    color = s.run(W, H, [(R.F_RGBA32F, None)])[0]
    s = R.Shader.get("motion_blur", samples=int(p.samples))  # MotionBlurEffect.update  src/motion-blur/MotionBlurEffect.js:87-102
    s.set(optional=("texSize",), intensity=float(p.intensity), jitter=float(p.jitter), deltaTime=float(p.delta_time), frame=int(p.frame),
          resolution=list(p.resolution))
    s.tex("velocityTexture", velocity, R.F_RGBA32F)
    s.tex("inputTexture", inp, R.F_RGBA16F, linear=True)
    s.tex("inputBuffer", color, R.F_RGBA32F)
    s.tex("blueNoiseTexture", blue_noise, R.F_RGBA8, repeat=True)
    s.set(blueNoiseSize=[blue_noise.shape[1], blue_noise.shape[0]], optional=("blueNoiseIndex",), blueNoiseIndex=0)
    return s.run(W, H, [(R.F_RGBA16F, None)])[0]


def reference_available(samples: int) -> bool:
    import refglsl as R

    return R.available("traa_compose") and R.available("motion_blur", samples=int(samples))


def digest(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def pins() -> dict:
    with open(PINS, encoding="utf-8") as f:
        return json.load(f)
