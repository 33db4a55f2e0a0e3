"""K6h, the horizon-march AO pass, on the CPU: the C++ oracle (tests/horizon_oracle.cpp) against an independent numpy fp32 restatement
of the definition in DESIGN.md §1 (K6h), known answers, the direction table, and the host surfaces (option table, ctypes layout, shim).

The restatement lowers every operation the way oracle/glsl.h and the kernels do: fp32 IEEE arithmetic, fma where glsl.h uses one
(emulated in float64: the product of two floats is exact there), vector / scalar as one reciprocal and multiplies."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import ao_harness as ao
import chain_harness as ch
import horizon_harness as hz
from realism_effects_b200 import abi, effects, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32, f64 = np.float32, np.float64


# ------------------------------------------------------------------------------------------------------------------ numpy restatement
def fma(a, b, c):
    return (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(f32)


def mat_vec(M, v):  # M * v, M column-major float32[16]
    x, y, z, w = v
    return [fma(M[r], x, fma(M[4 + r], y, fma(M[8 + r], z, (M[12 + r] * w).astype(f32)))) for r in range(4)]


def vec_mat(v, M):  # v * M
    x, y, z, w = v
    return [fma(x, M[4 * c], fma(y, M[4 * c + 1], fma(z, M[4 * c + 2], (w * M[4 * c + 3]).astype(f32)))) for c in range(4)]


def dot3(a, b):
    return fma(a[2], b[2], fma(a[1], b[1], (a[0] * b[0]).astype(f32)))


def cross3(a, b):
    return [fma(a[1], b[2], -(b[1] * a[2])), fma(a[2], b[0], -(b[2] * a[0])), fma(a[0], b[1], -(b[0] * a[1]))]


def scale3(a, s):
    return [(c * s).astype(f32) for c in a]


def normalize3(a):
    return scale3(a, (f32(1) / np.sqrt(dot3(a, a))).astype(f32))


def nearest(plane, u, v):  # NEAREST, clamp to edge
    h, w = plane.shape[:2]
    ix = np.clip(np.floor((u * f32(w)).astype(f32)).astype(np.int64), 0, w - 1)
    iy = np.clip(np.floor((v * f32(h)).astype(f32)).astype(np.int64), 0, h - 1)
    return plane[iy, ix]


def world_pos(Pinv, Cmw, depth, u, v):  # hbao_utils.glsl:19-29
    one = np.ones_like(depth)
    clip = [(u * f32(2) - f32(1)).astype(f32), (v * f32(2) - f32(1)).astype(f32), (depth * f32(2) - f32(1)).astype(f32), one]
    ws = mat_vec(Cmw, mat_vec(Pinv, clip))
    return scale3(ws[:3], (f32(1) / ws[3]).astype(f32))


def world_normal(Pinv, Cmw, View, depth, normal, u, v):
    if normal is not None:
        t = nearest(normal, u, v).astype(f32)
        n = [((t[..., i] / f32(255)).astype(f32) * f32(2) - f32(1)).astype(f32) for i in range(3)]
        return normalize3(vec_mat(n + [np.ones_like(u)], View)[:3])
    DH, DW = depth.shape
    sx, sy = f32(DW), f32(DH)
    ix, iy = (u * sx).astype(f32).astype(np.int64), (v * sy).astype(f32).astype(np.int64)

    def D(dx, dy):
        return depth[np.clip(iy + dy, 0, DH - 1), np.clip(ix + dx, 0, DW - 1)]

    c0, l2, l1, r1, r2, b2, b1, t1, t2 = D(0, 0), D(-2, 0), D(-1, 0), D(1, 0), D(2, 0), D(0, -2), D(0, -1), D(0, 1), D(0, 2)

    def dev(n1, n2):
        return np.abs(((f32(2) * n1).astype(f32) - n2) - c0).astype(f32)

    dl, dr, db, dt = dev(l1, l2), dev(r1, r2), dev(b1, b2), dev(t1, t2)
    ce = world_pos(Pinv, Cmw, c0, u, v)
    ox, oy = f32(1) / sx, f32(1) / sy
    L, R = world_pos(Pinv, Cmw, l1, (u - ox).astype(f32), v), world_pos(Pinv, Cmw, r1, (u + ox).astype(f32), v)
    B, T = world_pos(Pinv, Cmw, b1, u, (v - oy).astype(f32)), world_pos(Pinv, Cmw, t1, u, (v + oy).astype(f32))
    dpdx = [np.where(dl < dr, ce[i] - L[i], -ce[i] + R[i]).astype(f32) for i in range(3)]
    dpdy = [np.where(db < dt, ce[i] - B[i], -ce[i] + T[i]).astype(f32) for i in range(3)]
    return normalize3(cross3(dpdx, dpdy))


def blue_shift(index: int, size: int):
    """pcg4d of rng_initialize (blue_noise.glsl:13-34) in uint32 arithmetic: the texel shift of blue-noise index `index`"""
    m = 0xFFFFFFFF
    ui = index & m
    v = [ui, (ui * 15843) & m, (ui * 31 + 4566) & m, (ui * 2345 + 58585) & m]
    v = [(x * 1664525 + 1013904223) & m for x in v]

    def mix(v):
        v[0] = (v[0] + v[1] * v[3]) & m
        v[1] = (v[1] + v[2] * v[0]) & m
        v[2] = (v[2] + v[0] * v[1]) & m
        v[3] = (v[3] + v[1] * v[2]) & m

    mix(v)
    v = [x ^ (x >> 16) for x in v]
    mix(v)
    return (v[0] % 0x0FFFFFFF) % size, (v[1] % 0x0FFFFFFF) % size


def directions_table(D: int) -> np.ndarray:
    out = np.zeros((D, 256, 2), np.float32)
    for d in range(D):
        for b in range(256):
            theta = 2.0 * math.pi * (d + b / 255.0) / D
            out[d, b] = (math.cos(theta), math.sin(theta))
    return out


def numpy_horizon(p: abi.HbaoHorizonParams, depth, blue, out_prev, normal=None, branches: dict | None = None):
    """DESIGN.md §1 K6h, restated; returns the RGBA16F target.  `branches`, if given, receives per-pixel masks of the branches the
    pixel takes: foreground, r_px < 1, the max_radius_pixels clamp binding, and the final clamp saturating at 0 and at 1."""
    H, W = out_prev.shape[:2]
    M = {k: np.asarray(getattr(p, k)[:], f32) for k in ("projection", "projection_inverse", "camera_matrix_world", "view_matrix")}
    Proj, Pinv, Cmw, View = M["projection"], M["projection_inverse"], M["camera_matrix_world"], M["view_matrix"]
    rx, ry = (f32(W), f32(H)) if (p.resolution[0], p.resolution[1]) == (0.0, 0.0) else (f32(p.resolution[0]), f32(p.resolution[1]))
    xs, ys = np.meshgrid(np.arange(W, dtype=f32), np.arange(H, dtype=f32))
    u, v = ((xs + f32(0.5)) / f32(W)).astype(f32), ((ys + f32(0.5)) / f32(H)).astype(f32)
    depth = np.asarray(depth, f32)
    d0 = nearest(depth, u, v)
    P = world_pos(Pinv, Cmw, d0, u, v)
    N = world_normal(Pinv, Cmw, View, depth, normal, u, v)
    one = np.ones_like(u)
    vs = mat_vec(Pinv, [(u * f32(2) - f32(1)).astype(f32), (v * f32(2) - f32(1)).astype(f32), (d0 * f32(2) - f32(1)).astype(f32), one])
    Pv = scale3(vs[:3], (f32(1) / vs[3]).astype(f32))
    w_clip = mat_vec(Proj, Pv + [one])[3]
    r_px = ((((f32(p.distance) * f32(0.5)).astype(f32) * ry).astype(f32) * Proj[5]).astype(f32) / w_clip).astype(f32)
    delta = (np.minimum(r_px, f32(p.max_radius_pixels)) / f32(p.steps + 1)).astype(f32)
    sx, sy = blue_shift(p.blue_noise_index, blue.shape[0])
    bx, by = (u * rx).astype(f32).astype(np.int64), (v * ry).astype(f32).astype(np.int64)
    texel = blue[(by + sy) % blue.shape[0], (bx + sx) % blue.shape[1]]
    br, j = texel[..., 0].astype(np.int64), (texel[..., 1].astype(f32) / f32(255)).astype(f32)
    table = directions_table(p.directions)
    dist2 = f32(p.distance) * f32(p.distance)
    s = np.zeros_like(u)
    for d in range(p.directions):
        dx, dy = table[d, br, 0], table[d, br, 1]
        for k in range(p.steps):
            t = (f32(1) + ((f32(k) + j).astype(f32) * delta).astype(f32)).astype(f32)
            ox = np.floor((dx * t).astype(f32) + f32(0.5)).astype(f32)
            oy = np.floor((dy * t).astype(f32) + f32(0.5)).astype(f32)
            su, sv = (u + (ox / rx).astype(f32)).astype(f32), (v + (oy / ry).astype(f32)).astype(f32)
            Q = world_pos(Pinv, Cmw, nearest(depth, su, sv), su, sv)
            V = [(Q[i] - P[i]).astype(f32) for i in range(3)]
            vv = dot3(V, V)
            pos = vv > 0
            safe = np.where(pos, vv, f32(1))
            c = np.clip((dot3(N, V) / np.sqrt(safe)).astype(f32) - f32(p.angle_bias), 0, 1).astype(f32)
            f = np.clip(f32(1) - (safe / dist2).astype(f32), 0, 1).astype(f32)
            s = (s + np.where(pos, (c * f).astype(f32), f32(0))).astype(f32)
    ao_raw = (f32(1) - ((f32(p.intensity) * s).astype(f32) / f32(p.directions * p.steps)).astype(f32)).astype(f32)
    ao = np.where(r_px >= f32(1), np.clip(ao_raw, 0, 1).astype(f32), f32(1))
    out = np.array(out_prev, np.float16, copy=True)
    fg = d0 != f32(1)
    if branches is not None:
        marched = fg & (r_px >= f32(1))
        branches.update(fg=fg, radius_under_one=fg & (r_px < f32(1)), clamp_binds=marched & (r_px > f32(p.max_radius_pixels)),
                        clamp_free=marched & (r_px <= f32(p.max_radius_pixels)), saturate_0=marched & (ao_raw <= 0), saturate_1=marched & (ao_raw >= 1))
    out[fg] = np.stack(N + [ao], -1)[fg].astype(np.float16)
    return out


# ------------------------------------------------------------------------------------------------------------------ option grid
# The scenes of tests/test_gpu_horizon_ao.py: (width, height, orthographic, resolutionScale).  201 x 121 at 0.5 has the fractional
# `resolution` (100.5, 60.5) over a 100 x 60 target.
HZ_SCENES = ((200, 120, False, 1.0), (201, 121, False, 0.5), (200, 120, True, 1.0))
# a distance at which some foreground pixels have r_px < 1 and the others march (perspective); the orthographic r_px is one value for the
# whole frame, so there it is under 1 everywhere
SMALL_DISTANCE = {(200, 120, False, 1.0): 0.15, (201, 121, False, 0.5): 0.3, (200, 120, True, 1.0): 0.15}
LARGE_DISTANCE = 50.0  # the max_radius_pixels clamp binds on most pixels


class HzCase:
    def __init__(self, scene, distance=2.0, max_radius_pixels=64.0, angle_bias=0.1, intensity=1.0):
        self.scene, self.distance, self.max_radius_pixels, self.angle_bias, self.intensity = scene, distance, max_radius_pixels, angle_bias, intensity

    def __str__(self):
        W, H, ortho, scale = self.scene
        return (f"{W}x{H}{'-ortho' if ortho else ''}-s{scale}-d{self.distance:g}-mr{self.max_radius_pixels:g}-ab{self.angle_bias:g}"
                f"-i{self.intensity:g}")

    def params(self, cam_u: dict, res, index: int = 4711) -> abi.HbaoHorizonParams:
        return hz.horizon_params(cam_u, index, 8, 32, res, distance=self.distance, angle_bias=self.angle_bias, intensity=self.intensity,
                                 max_radius_pixels=self.max_radius_pixels)


def _hz_grid() -> list:
    out = []
    for sc in HZ_SCENES:
        small = SMALL_DISTANCE[sc]
        out += [HzCase(sc), HzCase(sc, distance=small), HzCase(sc, distance=LARGE_DISTANCE), HzCase(sc, max_radius_pixels=1.0),
                HzCase(sc, max_radius_pixels=7.5), HzCase(sc, angle_bias=0.0), HzCase(sc, angle_bias=0.9), HzCase(sc, intensity=0.0),
                HzCase(sc, intensity=16.0), HzCase(sc, LARGE_DISTANCE, 7.5, 0.0, 16.0), HzCase(sc, small, 1.0, 0.9, 16.0)]
    return out


HZ_CASES = _hz_grid()


def hz_inputs(scene, cache: dict = {}):  # noqa: B006  (one set of frames per scene for the whole session)
    if scene not in cache:
        W, H, ortho, _ = scene
        cache[scene] = ch.make_inputs(W, H, 2, orthographic=ortho)
    return cache[scene]


def hz_call(case: HzCase):
    """(params, depth, blue noise, target filled with a sentinel) of `case` on frame 1 of its scene"""
    W, H, _, scale = case.scene
    inp = hz_inputs(case.scene)
    f1 = inp.frames[1]
    (tw, th), res = ao.ao_target_size(W, H, scale)
    return case.params(f1["cam"], res), f1["depth"], inp.blue, np.full((th, tw, 4), -3.0, np.float16)


def test_option_grid_reaches_every_branch():
    """the K6h option grid of tests/test_gpu_horizon_ao.py, counted with the numpy restatement: on each perspective scene one case has
    pixels with r_px < 1 (AO 1) beside pixels that march; on each scene the max_radius_pixels clamp binds on most pixels of one case and
    on none of another; the final clamp saturates at 0 and at 1"""
    for sc in HZ_SCENES:
        counts = []
        for case in (c for c in HZ_CASES if c.scene == sc):
            p, depth, blue, prev = hz_call(case)
            b = {}
            numpy_horizon(p, depth, blue, prev, branches=b)
            counts.append((case, {k: float(v.sum() / b["fg"].sum()) for k, v in b.items() if k != "fg"}))
        name = str(counts[0][0])
        if sc[2]:
            assert any(c["radius_under_one"] == 1.0 for _, c in counts), name
        else:
            assert any(0.05 < c["radius_under_one"] < 0.95 for _, c in counts), (name, counts)
        assert any(c["clamp_binds"] > 0.5 for case, c in counts if case.distance == LARGE_DISTANCE), name
        assert any(c["clamp_binds"] == 0.0 and c["clamp_free"] > 0.9 for _, c in counts), name
        assert any(c["clamp_binds"] > 0.9 for case, c in counts if case.max_radius_pixels == 7.5), name
        assert any(c["saturate_0"] > 0 for _, c in counts), name
        assert any(0 < c["saturate_1"] < 1 for _, c in counts) and any(c["saturate_1"] == 1.0 for case, c in counts if case.intensity == 0), name


# ------------------------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def frames():
    return {ortho: ch.make_inputs(64, 48, 2, orthographic=ortho) for ortho in (False, True)}


@pytest.mark.parametrize("directions,steps", [(1, 1), (1, 32), (8, 1), (8, 32), (32, 1), (32, 32)])
@pytest.mark.parametrize("with_normal", [False, True])
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("ortho", [False, True])
def test_oracle_equals_numpy_restatement(frames, directions, steps, with_normal, scale, ortho):
    inp = frames[ortho]
    f1 = inp.frames[1]
    (tw, th), res = ao.ao_target_size(64, 48, scale)
    normal = ao.view_normal_plane(64, 48, 1, f1["cam"]) if with_normal else None
    p = hz.horizon_params(f1["cam"], 4711, directions, steps, res)
    prev = np.full((th, tw, 4), -7.0, np.float16)
    want = numpy_horizon(p, f1["depth"], inp.blue, prev, normal)
    got = hz.oracle_hbao_horizon(p, f1["depth"], inp.blue, prev, normal=normal)
    diff = (want.view(np.uint16) != got.view(np.uint16)).any(-1)
    assert diff.sum() == 0, f"{diff.sum()} pixels differ"
    a = got[..., 3].astype(np.float32)
    fg = a != -7
    assert fg.any() and (a[fg] < 1).any(), "the synthetic frame must occlude somewhere"


def test_direction_table_is_deterministic_and_shared(built):
    """the host's table (librfx, built once per `directions` value) equals the oracle's and a Python-libm evaluation of the same formula"""
    for D in (1, 3, 8, 32):
        host = np.zeros((D, 256, 2), np.float32)
        assert abi.lib().rfx_hbao_horizon_directions(D, host.ctypes.data) == 0
        assert np.array_equal(host.view(np.uint32), hz.oracle_directions(D).view(np.uint32))
        assert np.array_equal(host.view(np.uint32), directions_table(D).view(np.uint32))
    for bad in (0, 33, -1):
        assert abi.lib().rfx_hbao_horizon_directions(bad, np.zeros(2 * 256 * 40, np.float32).ctypes.data) != 0


# ------------------------------------------------------------------------------------------------------------------ known answers
def ortho_camera(W: int, H: int, texel: float = 0.1, near: float = 0.1, far: float = 10.0) -> dict:
    """an orthographic camera at the origin looking down -z, `texel` world units per pixel"""
    right, top = W * texel / 2, H * texel / 2
    P = np.zeros((4, 4))
    P[0, 0], P[1, 1], P[2, 2], P[2, 3], P[3, 3] = 1 / right, 1 / top, -2 / (far - near), -(far + near) / (far - near), 1
    eye = np.eye(4).T.reshape(16).astype(np.float32)
    return dict(projection=P.T.reshape(16).astype(np.float32), projection_inverse=np.linalg.inv(P).T.reshape(16).astype(np.float32),
                camera_matrix_world=eye, view_matrix=eye, near=near, far=far)


def ortho_depth(view_z, near=0.1, far=10.0):
    return np.asarray((-view_z - near) / (far - near), np.float32)  # viewZToOrthographicDepth


def test_plane_facing_the_camera_is_unoccluded(frames):
    inp = frames[False]
    cam = inp.frames[1]["cam"]
    depth = np.full((48, 64), 0.97, np.float32)
    for D, S in ((8, 32), (32, 8)):
        p = hz.horizon_params(cam, 99, D, S)
        out = hz.oracle_hbao_horizon(p, depth, inp.blue, np.zeros((48, 64, 4), np.float16))
        assert (out[..., 3] == 1).all()


def test_radius_under_one_texel_gives_one(frames):
    inp = frames[False]
    f1 = inp.frames[1]
    p = hz.horizon_params(f1["cam"], 99, 8, 32, distance=1e-4)
    prev = np.zeros((48, 64, 4), np.float16)
    out = hz.oracle_hbao_horizon(p, f1["depth"], inp.blue, prev)
    fg = f1["depth"] != 1
    assert (out[..., 3][fg] == 1).all()
    assert np.array_equal(out.view(np.uint16), numpy_horizon(p, f1["depth"], inp.blue, prev).view(np.uint16))


def test_concave_step_occludes_its_inner_edge_only():
    """a far plane (left) meeting a nearer block (right) at x = 32: the far plane's texels next to the step are occluded, those farther
    than the projected radius and every texel of the block are not"""
    W, H = 64, 48
    cam = ortho_camera(W, H)
    z = np.where(np.arange(W)[None, :] < 32, -5.0, -4.5) * np.ones((H, 1))
    depth = ortho_depth(z)
    blue = synth.load_blue_noise()
    p = hz.horizon_params(cam, 1234, 8, 16, distance=1.0)  # r_px = 1 * 0.5 * 48 / 2.4 = 10 texels
    out = hz.oracle_hbao_horizon(p, depth, blue, np.zeros((H, W, 4), np.float16)).astype(np.float32)
    a = out[..., 3]
    assert (a[:, 28:32] < 1).all(), a[:, 26:34]
    assert (a[:, :20] == 1).all() and (a[:, 32:] == 1).all()
    assert np.allclose(out[..., :3], [0, 0, 1], atol=1e-3)
    assert np.array_equal(out.astype(np.float16).view(np.uint16), numpy_horizon(p, depth, blue, np.zeros((H, W, 4), np.float16)).view(np.uint16))


def test_background_texels_are_left_untouched(frames):
    inp = frames[False]
    f1 = inp.frames[1]
    depth = f1["depth"].copy()
    depth[:, :20] = 1.0
    prev = np.full((48, 64, 4), 3.5, np.float16)
    out = hz.oracle_hbao_horizon(hz.horizon_params(f1["cam"], 5, 4, 8), depth, inp.blue, prev)
    bg = depth == 1
    assert bg[:, :20].all() and np.array_equal(out[bg].view(np.uint16), prev[bg].view(np.uint16))
    assert not np.array_equal(out[~bg].view(np.uint16), prev[~bg].view(np.uint16))


# ------------------------------------------------------------------------------------------------------------------ host surfaces
def test_option_table_and_js_literal_agree():
    t = effects.defaultHorizonAOOptions
    for k in ("directions", "steps", "angleBias", "intensity", "maxRadiusPixels", "resolutionScale", "distance", "power", "color", "useNormalPass",
              "velocityDepthNormalPass", "normalTexture", *effects.defaultPoissonBlurOptions):
        assert k in t, k
    for k in ("spp", "distancePower", "bias", "thickness"):
        assert k not in t, k
    assert (t["directions"], t["steps"], t["angleBias"], t["intensity"], t["maxRadiusPixels"]) == (8, 32, 0.1, 1, 64)
    js = open(os.path.join(ROOT, "js", "index.js"), encoding="utf-8").read()
    m = re.search(r"export const defaultHorizonAOOptions\s*=\s*\{(.*?)\n\}", js, flags=re.S)
    assert m, "js/index.js lacks defaultHorizonAOOptions"
    body = m.group(1)
    assert "...defaultPoissonBlurOptions" in body
    for k, v in t.items():
        if k in effects.defaultPoissonBlurOptions:
            continue
        lit = ("true" if v is True else "false" if v is False else "null" if v is None else "[0, 0, 0]" if k == "color" else "%g" % v)
        assert re.search(r"\b" + k + r":\s*" + re.escape(lit), body), (k, lit)
    for k in ("spp", "distancePower", "bias", "thickness"):
        assert not re.search(r"\b" + k + r":", body), k
    assert "export class HorizonAOEffect" in js


@pytest.mark.parametrize("key,bad", [("directions", 0), ("directions", 33), ("directions", 2.5), ("steps", 0), ("steps", 65), ("angleBias", -0.1),
                                     ("angleBias", 1.0), ("intensity", -1), ("maxRadiusPixels", 0.5), ("distance", 0), ("resolutionScale", 0),
                                     ("resolutionScale", 1.5)])
def test_out_of_range_options_raise(key, bad):
    with pytest.raises(abi.RfxError):
        effects.check_horizon_ao_options({**effects.defaultHorizonAOOptions, key: bad})
    effects.check_horizon_ao_options(dict(effects.defaultHorizonAOOptions))


def test_ctypes_layout_of_horizon_params_matches_c(tmp_path):
    src = tmp_path / "sz.c"
    fields = [f[0] for f in abi.HbaoHorizonParams._fields_]
    body = "".join(f'printf("{f} %zu\\n", offsetof(rfx_hbao_horizon_params, {f}));' for f in fields)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rfx.h"\n'
                   f'int main(void){{printf("size %zu\\n", sizeof(rfx_hbao_horizon_params));{body} return 0;}}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out["size"]) == C.sizeof(abi.HbaoHorizonParams) and C.sizeof(abi.HbaoHorizonParams) % 16 == 0
    for f in fields:
        assert int(out[f]) == getattr(abi.HbaoHorizonParams, f).offset, f


def test_shim_binds_hbao_horizon():
    shim = open(os.path.join(ROOT, "js", "napi", "shim.cc"), encoding="utf-8").read()
    assert re.search(r'FN\("hbaoHorizon",\s*HbaoHorizon\)', shim)
    assert "rfx_hbao_horizon_launch(" in shim
    js = open(os.path.join(ROOT, "js", "index.js"), encoding="utf-8").read()
    assert "rfx.hbaoHorizon(" in js
    r = subprocess.run(["bash", os.path.join(ROOT, "tools", "check_shim.sh")], capture_output=True, text=True)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr
