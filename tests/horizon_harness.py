"""K6h, the horizon-march AO pass — TEST INFRASTRUCTURE.

* `oracle_hbao_horizon`: tests/horizon_oracle.cpp (the CPU oracle of oracle/rfx_oracle.cpp and tests/ao_oracle.cpp extended by K6h),
  bound with ctypes and built on first use into build/ (git-ignored) with oracle/Makefile's flags.
* `oracle_directions`: the direction table the oracle builds.
* `horizon_params`: rfx_hbao_horizon_params for a camera of chain_harness.make_inputs, with HorizonAOEffect's defaults.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from realism_effects_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "horizon_oracle.cpp")
SO = os.path.join(ROOT, "build", "librfx_oracle_horizon.so")
_DEPS = [SRC, os.path.join(ROOT, "tests", "ao_oracle.cpp"), os.path.join(ROOT, "oracle", "rfx_oracle.cpp"), os.path.join(ROOT, "oracle", "glsl.h"),
         os.path.join(ROOT, "oracle", "Makefile"), os.path.join(ROOT, "include", "rfx.h")]
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wall", "-Wno-unused-function",
            "-Wno-unused-variable", "-Wno-unused-but-set-variable"]  # oracle/Makefile's CXXFLAGS


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


def oracle_directions(directions: int) -> np.ndarray:
    """(directions, 256, 2) float32: (cos, sin) of 2 pi (d + b / 255) / directions"""
    out = np.zeros((directions, 256, 2), np.float32)
    _L().orc_horizon_directions(C.c_int(directions), _p(out))
    return out


def oracle_hbao_horizon(p: abi.HbaoHorizonParams, depth, blue_noise, out_prev, *, normal=None) -> np.ndarray:
    """K6h on the CPU.  out_prev (H, W, 4) float16 is the AO target before the pass (its size is the target's); background texels keep it."""
    DH, DW = depth.shape
    out = np.array(np.ascontiguousarray(out_prev).view(np.uint16), copy=True)
    H, W = out.shape[:2]
    bn = np.ascontiguousarray(blue_noise, np.uint8)
    n = None if normal is None else np.ascontiguousarray(normal, np.uint8)
    assert n is None or n.shape[:2] == (DH, DW)
    _L().orc_ao_hbao_horizon(C.byref(p), C.c_int(W), C.c_int(H), _p(np.ascontiguousarray(depth, np.float32)), C.c_int(DW), C.c_int(DH), _p(n), _p(bn),
                             C.c_int(bn.shape[1]), C.c_int(bn.shape[0]), _p(out))
    return out.view(np.float16)


def horizon_params(cam_u: dict, index: int, directions: int = 8, steps: int = 32, resolution=None, *, distance: float = 2.0, angle_bias: float = 0.1,
                   intensity: float = 1.0, max_radius_pixels: float = 64.0) -> abi.HbaoHorizonParams:
    """HorizonAOEffect's defaults (effects.defaultHorizonAOOptions); resolution None = {0, 0}, the target's own size"""
    p = abi.HbaoHorizonParams()
    for k in ("projection", "projection_inverse", "camera_matrix_world", "view_matrix"):
        abi.set_f16(getattr(p, k), cam_u[k])
    if resolution is not None:
        p.resolution[:] = [float(resolution[0]), float(resolution[1])]
    p.distance, p.angle_bias, p.intensity, p.max_radius_pixels = distance, angle_bias, intensity, max_radius_pixels
    p.directions, p.steps, p.blue_noise_index = directions, steps, index
    return p
