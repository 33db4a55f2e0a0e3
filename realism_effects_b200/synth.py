"""Deterministic synthetic inputs for the hot path (SURVEY.md §8d).

An analytic "Sponza-like" scene (floor, two side walls, back wall, a 4x2 grid of box columns,
one sphere, open ceiling => background pixels) is ray-cast per pixel and written out *in the
reference's plane formats*:

  gBuffer  RGBA32F  packGBuffer()            src/gbuffer/shader/gbuffer_packing.glsl:166-178
  depth    R32F     NDC depth, 1.0 = background (src/gbuffer/GBufferPass.js:42-44)
  velocity RGBA32F  (uv motion, packed oct normal, depth)
                    src/temporal-reproject/material/VelocityDepthNormalMaterial.js:76-83,186-188
  direct   RGBA16F  albedo * max(n.L, 0)     (composer input buffer, example/main.js:173)

Camera math follows three.js (PerspectiveCamera.updateProjectionMatrix, Matrix4.lookAt /
compose / invert) so the matrices handed to the kernels are the ones a three.js host would
upload.  Everything is computed with torch so the same code runs on the CPU (tests, golden
fixtures) and on the GPU (bench.py input generation).  This module is NOT on the hot path and
does not touch `oracle/`.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field

import numpy as np
import torch

# --------------------------------------------------------------------------------------
# three.js camera math (float64, then rounded to float32 like a Float32Array uniform upload)
# --------------------------------------------------------------------------------------


def perspective_matrix(fov_deg: float, aspect: float, near: float, far: float) -> np.ndarray:
    """three.js PerspectiveCamera.updateProjectionMatrix + Matrix4.makePerspective (row-major 4x4)."""
    top = near * math.tan(math.radians(0.5 * fov_deg))
    height = 2 * top
    width = aspect * height
    left = -0.5 * width
    right, bottom = left + width, top - height
    x = 2 * near / (right - left)
    y = 2 * near / (top - bottom)
    a = (right + left) / (right - left)
    b = (top + bottom) / (top - bottom)
    c = -(far + near) / (far - near)
    d = -2 * far * near / (far - near)
    return np.array([[x, 0, a, 0], [0, y, b, 0], [0, 0, c, d], [0, 0, -1, 0]], dtype=np.float64)


def look_at_world_matrix(eye, target, up=(0.0, 1.0, 0.0)) -> np.ndarray:
    """camera.matrixWorld for camera.position=eye; camera.lookAt(target) (row-major 4x4)."""
    eye = np.asarray(eye, np.float64)
    z = eye - np.asarray(target, np.float64)
    z /= np.linalg.norm(z)
    x = np.cross(np.asarray(up, np.float64), z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = x, y, z, eye
    return m


def col_major32(m: np.ndarray) -> np.ndarray:
    """row-major 4x4 float64 -> 16 float32 in three.js (column-major) element order."""
    return np.ascontiguousarray(m.T.reshape(16)).astype(np.float32)


@dataclass
class Camera:
    """A three.js PerspectiveCamera snapshot."""

    fov: float = 40.0
    aspect: float = 16 / 9
    near: float = 0.01
    far: float = 250.0
    position: tuple = (0.0, 8.75, 25.0)
    target: tuple = (0.0, 8.75, 0.0)
    proj: np.ndarray = field(init=False)
    world: np.ndarray = field(init=False)

    def __post_init__(self):
        self.view_offset = None  # three.js camera.view (setViewOffset): sub-pixel TRAA jitter
        self.updateProjectionMatrix()
        self.world = look_at_world_matrix(self.position, self.target)

    # -- three.js PerspectiveCamera.setViewOffset / clearViewOffset / updateProjectionMatrix -----------------------------------
    def setViewOffset(self, fullWidth, fullHeight, x, y, width, height):
        self.view_offset = dict(enabled=True, fullWidth=fullWidth, fullHeight=fullHeight, offsetX=x, offsetY=y, width=width, height=height)
        self.updateProjectionMatrix()

    def clearViewOffset(self):
        if self.view_offset is not None:
            self.view_offset["enabled"] = False
        self.updateProjectionMatrix()

    def updateProjectionMatrix(self):
        near = self.near
        top = near * math.tan(math.radians(0.5 * self.fov))
        height = 2 * top
        width = self.aspect * height
        left = -0.5 * width
        v = self.view_offset
        if v is not None and v["enabled"]:
            left += v["offsetX"] * width / v["fullWidth"]
            top -= v["offsetY"] * height / v["fullHeight"]
            width *= v["width"] / v["fullWidth"]
            height *= v["height"] / v["fullHeight"]
        right, bottom, far = left + width, top - height, self.far
        x, y = 2 * near / (right - left), 2 * near / (top - bottom)
        a, b = (right + left) / (right - left), (top + bottom) / (top - bottom)
        c, d = -(far + near) / (far - near), -2 * far * near / (far - near)
        self.proj = np.array([[x, 0, a, 0], [0, y, b, 0], [0, 0, c, d], [0, 0, -1, 0]], dtype=np.float64)

    def unjittered_uniforms(self) -> dict:
        """uniforms with camera.view disabled, as TemporalReprojectPass.render uploads them (TemporalReprojectPass.js:168-186)"""
        v, saved = self.view_offset, self.proj
        if v is not None and v["enabled"]:
            v["enabled"] = False
            self.updateProjectionMatrix()
            u = self.uniforms()
            v["enabled"] = True
            self.proj = saved
            return u
        return self.uniforms()

    @property
    def view(self):
        return np.linalg.inv(self.world)

    @property
    def proj_inv(self):
        return np.linalg.inv(self.proj)

    def uniforms(self) -> dict:
        """float32 column-major arrays as a three.js host would upload them."""
        return dict(
            projection=col_major32(self.proj),
            projection_inverse=col_major32(self.proj_inv),
            camera_matrix_world=col_major32(self.world),
            view_matrix=col_major32(self.view),
            near=np.float32(self.near),
            far=np.float32(self.far),
            position=np.asarray(self.position, np.float32),
        )


# --------------------------------------------------------------------------------------
# the reference's packers, restated with torch (bit-exact integer / half arithmetic)
# --------------------------------------------------------------------------------------
NON_ZERO_OFFSET = 0.0001
ONE_SAFE = 0.999999


def _f32(x):
    return x.to(torch.float32)


def pack_half2x16(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """packHalf2x16(vec2(a,b)) reinterpreted as float32 (uintBitsToFloat)."""
    ha = _f32(a).to(torch.float16).view(torch.int16).to(torch.int32) & 0xFFFF
    hb = _f32(b).to(torch.float16).view(torch.int16).to(torch.int32) & 0xFFFF
    return (ha | (hb << 16)).view(torch.float32)


def encode_oct_wrap(n: torch.Tensor):
    """gbuffer_packing.glsl:36-50 ; n: (...,3) float32"""
    n = n / (n[..., 0].abs() + n[..., 1].abs() + n[..., 2].abs()).unsqueeze(-1)
    x, y, z = n[..., 0], n[..., 1], n[..., 2]
    wx = 1.0 - y.abs()
    wy = 1.0 - x.abs()
    wx = torch.where(x < 0, -wx, wx)
    wy = torch.where(y < 0, -wy, wy)
    ox = torch.where(z > 0, x, wx)
    oy = torch.where(z > 0, y, wy)
    return ox * 0.5 + 0.5, oy * 0.5 + 0.5


def pack_normal(n: torch.Tensor) -> torch.Tensor:
    ox, oy = encode_oct_wrap(_f32(n))
    return pack_half2x16(ox, oy)


def vec4_to_float(v: torch.Tensor) -> torch.Tensor:
    """gbuffer_packing.glsl:143-149 ; v: (...,4) float32 in [0,1]"""
    v = torch.clamp_max(_f32(v) + NON_ZERO_OFFSET, ONE_SAFE)
    q = (v * 255.0).to(torch.int32)  # uvec4(): truncation
    bits = (q[..., 3] << 24) | (q[..., 2] << 16) | (q[..., 1] << 8) | q[..., 0]
    return bits.view(torch.float32)


def color2float(rgb: torch.Tensor) -> torch.Tensor:
    """gbuffer_packing.glsl:17-22"""
    c = torch.clamp_max(_f32(rgb) + NON_ZERO_OFFSET, ONE_SAFE)
    p, p1 = 256.0, 257.0
    return (
        torch.floor(c[..., 0] * p + 0.5)
        + torch.floor(c[..., 2] * p + 0.5) * p1
        + torch.floor(c[..., 1] * p + 0.5) * p1 * p1
    )


def encode_rgbe8(rgb: torch.Tensor) -> torch.Tensor:
    """gbuffer_packing.glsl:127-134.  Zero radiance takes a NaN path in the reference
    (log2(0)); its decoded value is 0 on every back-end, so it is encoded here as (0,0,0,0)."""
    rgb = _f32(rgb)
    mx = rgb.max(dim=-1).values
    safe = torch.where(mx > 0, mx, torch.ones_like(mx))
    fexp = torch.ceil(torch.log2(safe))
    out = torch.cat([rgb / torch.exp2(fexp).unsqueeze(-1), ((fexp + 128.0) / 255.0).unsqueeze(-1)], dim=-1)
    return torch.where((mx > 0).unsqueeze(-1), out, torch.full_like(out, -1.0))  # -1 + 1e-4 < 0 -> uint 0


def pack_gbuffer(diffuse4, normal, roughness, metalness, emissive) -> torch.Tensor:
    """packGBuffer  gbuffer_packing.glsl:166-178  -> (...,4) float32"""
    r = vec4_to_float(diffuse4)
    g = pack_normal(normal)
    rm = torch.stack([_f32(roughness), _f32(metalness), torch.zeros_like(_f32(roughness))], dim=-1)
    b = color2float(rm)
    e = encode_rgbe8(emissive)
    e = torch.clamp_min(e, -NON_ZERO_OFFSET)  # keeps (v + offset) >= 0 so the uint conversion is defined
    a = vec4_to_float(e)
    return torch.stack([r, g, b, a], dim=-1)


# --------------------------------------------------------------------------------------
# scene
# --------------------------------------------------------------------------------------
LIGHT_DIR = (0.7299, 0.4540, 0.5111)  # example/main.js:175-179,336-341 (yaw 55deg, pitch 27deg)

# (min xyz, max xyz, roughness, metalness, emissive rgb, palette id)
_BOXES = [
    ((-12.0, -1.0, -15.0), (12.0, 0.0, 30.0), 0.3, 0.0, (0, 0, 0), 0),   # floor
    ((-13.0, 0.0, -15.0), (-12.0, 14.0, 30.0), 1.0, 0.0, (0, 0, 0), 1),  # left wall
    ((12.0, 0.0, -15.0), (13.0, 14.0, 30.0), 1.0, 0.0, (0, 0, 0), 1),    # right wall
    ((-13.0, 0.0, -16.0), (13.0, 14.0, -15.0), 0.6, 0.0, (0, 0, 0), 2),  # back wall
]
for _ix, _x in enumerate((-7.5, -2.5, 2.5, 7.5)):
    for _iz, _z in enumerate((-8.0, 2.0)):
        _rough = (0.05, 0.3, 0.6, 1.0)[(_ix + 2 * _iz) % 4]
        _metal = 1.0 if (_ix + _iz) % 2 == 0 else 0.0
        _emis = (2.0, 1.0, 0.5) if (_ix, _iz) == (1, 1) else (0, 0, 0)
        _BOXES.append(((_x - 0.8, 0.0, _z - 0.8), (_x + 0.8, 9.0, _z + 0.8), _rough, _metal, _emis, 3 + (_ix + _iz) % 3))
_SPHERE = ((0.0, 3.0, 9.0), 3.0, 0.05, 1.0, 5)  # centre, radius, roughness, metalness, palette

_PALETTE = torch.tensor(
    [
        [[200, 190, 170], [90, 80, 70], [150, 60, 50]],
        [[180, 60, 50], [160, 150, 140], [60, 70, 140]],
        [[60, 140, 70], [170, 170, 160], [120, 110, 60]],
        [[220, 210, 200], [120, 120, 130], [200, 160, 60]],
        [[70, 90, 170], [210, 200, 190], [100, 100, 100]],
        [[230, 230, 230], [180, 150, 90], [140, 140, 150]],
    ],
    dtype=torch.float32,
)


@dataclass
class Frame:
    width: int
    height: int
    cam: Camera
    prev_cam: Camera
    depth: torch.Tensor         # (H,W)     f32
    gbuffer: torch.Tensor       # (H,W,4)   f32 (packed bits)
    velocity: torch.Tensor      # (H,W,4)   f32
    direct_light: torch.Tensor  # (H,W,4)   f16
    background: torch.Tensor    # (H,W) bool
    soa: dict | None = None     # the same frame as a conventional deferred renderer's planes (input of rfx_gbuffer_ingest_launch)


def render_frame(width: int, height: int, t: int = 0, *, device="cpu", cam_step=(0.02, 0.0, 0.0), static=False, fov: float = 40.0,
                 aspect: float | None = None, view_offset=None) -> Frame:
    """Ray-cast frame `t`.  The camera translates by `cam_step` per frame (SURVEY.md §8d); with
    `static=True` it does not move (exercises fullAccumulate).  `fov` = vertical field of view in degrees; `aspect`
    overrides width/height (non-square pixels: the same view sampled with more rows, used for weak scaling).
    `view_offset(camera, k)`, if given, is called on the camera of frame k (this frame's and the previous one) before anything is
    projected: a three.js setViewOffset, such as TRAA's sub-pixel jitter or a sub-rectangle of a larger frame (an off-axis frustum)."""
    aspect = width / height if aspect is None else aspect
    step = (0.0, 0.0, 0.0) if static else cam_step

    def cam_at(k):
        off = tuple(s * k for s in step)
        c = Camera(fov=fov, aspect=aspect, position=(0.0 + off[0], 8.75 + off[1], 25.0 + off[2]), target=(0.0 + off[0], 8.75 + off[1], 0.0 + off[2]))
        if view_offset is not None:
            view_offset(c, k)
        return c

    cam, prev = cam_at(t), cam_at(max(t - 1, 0))
    dev = torch.device(device)
    f64 = torch.float64
    xs = (torch.arange(width, device=dev, dtype=f64) + 0.5) / width * 2 - 1
    ys = (torch.arange(height, device=dev, dtype=f64) + 0.5) / height * 2 - 1
    ndc_y, ndc_x = torch.meshgrid(ys, xs, indexing="ij")
    pinv = torch.tensor(cam.proj_inv, device=dev, dtype=f64)
    world = torch.tensor(cam.world, device=dev, dtype=f64)
    # ray through the pixel centre (view space dir = projInv * (x, y, -1, 1))
    clip = torch.stack([ndc_x, ndc_y, -torch.ones_like(ndc_x), torch.ones_like(ndc_x)], dim=-1)
    vdir = clip @ pinv.T
    vdir = vdir[..., :3] / vdir[..., 3:4]
    vdir = vdir / vdir.norm(dim=-1, keepdim=True)
    d = vdir @ world[:3, :3].T
    o = world[:3, 3]

    best_t = torch.full((height, width), float("inf"), device=dev, dtype=f64)
    best_id = torch.full((height, width), -1, device=dev, dtype=torch.int64)
    normal = torch.zeros((height, width, 3), device=dev, dtype=f64)
    inv_d = 1.0 / torch.where(d.abs() < 1e-12, torch.full_like(d, 1e-12), d)
    for i, (bmin, bmax, *_rest) in enumerate(_BOXES):
        bmin_t = torch.tensor(bmin, device=dev, dtype=f64)
        bmax_t = torch.tensor(bmax, device=dev, dtype=f64)
        t0 = (bmin_t - o) * inv_d
        t1 = (bmax_t - o) * inv_d
        tn = torch.minimum(t0, t1)
        tf = torch.maximum(t0, t1)
        tnear, axis = tn.max(dim=-1)
        tfar = tf.min(dim=-1).values
        hit = (tnear < tfar) & (tnear > 1e-6) & (tnear < best_t)
        n = torch.zeros_like(d)
        sgn = -torch.sign(torch.gather(d, -1, axis.unsqueeze(-1))).squeeze(-1)
        n.scatter_(-1, axis.unsqueeze(-1), sgn.unsqueeze(-1))
        best_t = torch.where(hit, tnear, best_t)
        best_id = torch.where(hit, torch.full_like(best_id, i), best_id)
        normal = torch.where(hit.unsqueeze(-1), n, normal)
    sc, sr, s_rough, s_metal, s_pal = _SPHERE
    sc_t = torch.tensor(sc, device=dev, dtype=f64)
    oc = o - sc_t
    bq = (d * oc).sum(-1)
    cq = (oc * oc).sum(-1) - sr * sr
    disc = bq * bq - cq
    ts = -bq - torch.sqrt(torch.clamp_min(disc, 0))
    hit = (disc > 0) & (ts > 1e-6) & (ts < best_t)
    ps = o + ts.unsqueeze(-1) * d
    best_t = torch.where(hit, ts, best_t)
    best_id = torch.where(hit, torch.full_like(best_id, len(_BOXES)), best_id)
    normal = torch.where(hit.unsqueeze(-1), (ps - sc_t) / sr, normal)

    bg = best_id < 0
    tt = torch.where(bg, torch.ones_like(best_t), best_t)
    P = o + tt.unsqueeze(-1) * d
    P1 = torch.cat([P, torch.ones_like(P[..., :1])], dim=-1)

    def project(c: Camera):
        vp = torch.tensor(c.proj @ c.view, device=dev, dtype=f64)
        clipp = P1 @ vp.T
        return clipp

    c1 = project(cam)
    c0 = project(prev)
    depth = (0.5 * c1[..., 2] / c1[..., 3] + 0.5).to(torch.float32)  # fragCoordZ, VelocityDepthNormalMaterial.js:81
    depth = torch.where(bg, torch.ones_like(depth), torch.clamp(depth, 0.0, 0.99999994))
    pos1 = c1[..., :2] / c1[..., 3:4] * 0.5 + 0.5
    pos0 = c0[..., :2] / c0[..., 3:4] * 0.5 + 0.5
    vel = (pos1 - pos0).to(torch.float32)
    vel = torch.where(bg.unsqueeze(-1), torch.zeros_like(vel), vel)

    # materials
    n_obj = len(_BOXES) + 1
    rough_l = torch.tensor([b[2] for b in _BOXES] + [s_rough], device=dev, dtype=torch.float32)
    metal_l = torch.tensor([b[3] for b in _BOXES] + [s_metal], device=dev, dtype=torch.float32)
    emis_l = torch.tensor([b[4] for b in _BOXES] + [(0, 0, 0)], device=dev, dtype=torch.float32)
    pal_l = torch.tensor([b[5] for b in _BOXES] + [s_pal], device=dev, dtype=torch.int64)
    oid = torch.clamp_min(best_id, 0)
    cell = torch.floor(P * 0.5 + 1e-4).to(torch.int64)
    chk = (cell[..., 0] + cell[..., 1] + cell[..., 2]) % 3
    albedo = _PALETTE.to(dev)[pal_l[oid], chk] / 255.0  # 8-bit quantised
    roughness, metalness, emissive = rough_l[oid], metal_l[oid], emis_l[oid]
    nrm = normal.to(torch.float32)
    nrm = torch.where(bg.unsqueeze(-1), torch.tensor([0.0, 0.0, 1.0], device=dev), nrm)

    diffuse4 = torch.cat([albedo, torch.ones_like(albedo[..., :1])], dim=-1)
    gb = pack_gbuffer(diffuse4, nrm, roughness, metalness, emissive)
    clear = torch.tensor([0.0, 0.0, 0.0, 1.0], device=dev)  # cleared target (black, alpha 1)
    gb = torch.where(bg.unsqueeze(-1), clear, gb)

    velocity = torch.stack([vel[..., 0], vel[..., 1], pack_normal(nrm), depth], dim=-1)
    velocity = torch.where(bg.unsqueeze(-1), clear, velocity)  # background: (0,0,0,1)

    L = torch.tensor(LIGHT_DIR, device=dev, dtype=torch.float32)
    ndl = torch.clamp_min((nrm * L).sum(-1), 0.0)
    direct = albedo * (0.15 + 0.85 * ndl).unsqueeze(-1) + emissive
    sky = torch.tensor([0.35, 0.5, 0.8], device=dev)
    direct = torch.where(bg.unsqueeze(-1), sky, direct)
    direct4 = torch.cat([direct, torch.ones_like(direct[..., :1])], dim=-1).to(torch.float16)

    z1 = torch.zeros_like(nrm[..., :1])
    soa = dict(albedo=torch.round(diffuse4 * 255.0).to(torch.uint8).contiguous(),                       # RGBA8 (the palette is 8-bit)
               normal=torch.cat([nrm, z1], dim=-1).contiguous(),                                        # RGBA32F world normal
               material=torch.stack([roughness, metalness, torch.zeros_like(roughness), torch.zeros_like(roughness)], dim=-1).to(torch.float16).contiguous(),
               emissive=torch.cat([emissive, z1], dim=-1).to(torch.float16).contiguous(),
               motion=torch.cat([vel, z1, z1], dim=-1).contiguous())                                    # RGBA32F uv-space cur - prev
    return Frame(width, height, cam, prev, depth.contiguous(), gb.contiguous(), velocity.contiguous(), direct4.contiguous(), bg, soa)


# --------------------------------------------------------------------------------------
# environment map + importance-sampling tables
# --------------------------------------------------------------------------------------
def synthetic_env(width: int = 256, height: int = 128) -> np.ndarray:
    """An analytic HDR sky: horizon gradient + a bright sun lobe.  (H,W,4) float16, row 0 = v 0
    (the equirect `uv.y = 1 - acos(dir.y)/pi` convention => row 0 looks straight down)."""
    v = (np.arange(height) + 0.5) / height
    u = (np.arange(width) + 0.5) / width
    uu, vv = np.meshgrid(u, v)
    theta = (uu - 0.5) * 2 * np.pi
    phi = (1.0 - vv) * np.pi
    d = np.stack([np.sin(phi) * np.cos(theta), np.cos(phi), np.sin(phi) * np.sin(theta)], -1)
    up = np.clip(d[..., 1], 0, 1)
    sky = np.array([0.25, 0.45, 0.9]) * (0.3 + 0.7 * up[..., None]) + np.array([0.9, 0.8, 0.7]) * (1 - up[..., None]) ** 4 * 0.6
    ground = np.array([0.12, 0.1, 0.08])
    col = np.where((d[..., 1] > 0)[..., None], sky, ground)
    sun_dir = np.array(LIGHT_DIR) / np.linalg.norm(LIGHT_DIR)
    c = np.clip((d * sun_dir).sum(-1), 0, 1)
    col = col + np.array([60.0, 50.0, 40.0]) * (c[..., None] ** 400) + np.array([1.5, 1.2, 0.9]) * (c[..., None] ** 12)
    out = np.concatenate([col, np.ones_like(col[..., :1])], -1).astype(np.float16)
    return np.ascontiguousarray(out)


def build_env_cdf(data_f32: np.ndarray, flip_y: bool = False):
    """Restatement of `gatherData` (src/ssgi/utils/EquirectHdrInfoUniform.js:149-245), float32
    accumulators like the Float32Array code paths, float64 scalars where JS uses Numbers.
    data_f32: (H,W,4) float32 image memory.  Returns (marginal[H], conditional[H,W], totalSum).
    With flip_y the reference's in-place "un-flip" mirrors the top half over the bottom half (A4)."""
    data = np.array(data_f32, dtype=np.float32, copy=True)
    h, w = data.shape[:2]
    if flip_y:
        for y in range(h):  # y = 0..h-1 inclusive, in place  (:154-166)
            data[h - 1 - y] = data[y]
    lum = (0.2126 * data[..., 0].astype(np.float64) + 0.7152 * data[..., 1].astype(np.float64)) + 0.0722 * data[..., 2].astype(np.float64)  # JS: left to right
    cum64 = np.cumsum(lum, axis=1)                       # cumulativeRowWeight: a JS double accumulated left to right
    cdf_c = cum64.astype(np.float32)                     # cdfConditional[i] = cumulativeRowWeight (Float32Array store)
    row_sum = cum64[:, -1].copy()                        # the row's final cumulativeRowWeight (sequential, not a pairwise sum)
    total = float(np.cumsum(lum.reshape(-1))[-1])        # totalSumValue += weight, pixel after pixel in row-major order
    nz = row_sum != 0
    cdf_c[nz] = (cdf_c[nz].astype(np.float64) / row_sum[nz, None]).astype(np.float32)
    cdf_m = np.cumsum(row_sum)
    if cdf_m[-1] != 0:
        cdf_m = (cdf_m.astype(np.float32).astype(np.float64) / cdf_m[-1]).astype(np.float32)
    else:
        cdf_m = cdf_m.astype(np.float32)

    def closest(arr, target):  # binarySearchFindClosestIndexOf: first index with arr[i] >= target
        return min(int(np.searchsorted(arr, target, side="left")), len(arr) - 1)

    marginal = np.empty(h, np.float32)
    cdf_m64 = cdf_m.astype(np.float64)
    for i in range(h):
        marginal[i] = (closest(cdf_m64, (i + 1) / h) + 0.5) / h
    conditional = np.empty((h, w), np.float32)
    targets = (np.arange(w) + 1) / w
    for y in range(h):
        cols = np.minimum(np.searchsorted(cdf_c[y].astype(np.float64), targets, side="left"), w - 1)
        conditional[y] = (cols + 0.5) / w
    return marginal, conditional, total


def load_reference_env():
    """The reference demo's environment (example/public/hdr/spree_bank_1k.hdr, example/main.js:278; asset made by tools/make_env_asset.py),
    decoded the way three.js' RGBELoader decodes to HalfFloatType (RGBELoader.js: scale = 2^(e - 128) / 255, clamped to 65504, alpha 1).
    Returns (image_f16, gl_f16): `image_f16` (H, W, 4) float16 in image-memory order (top scanline first: what `gatherData` reads, with
    texture.flipY = true) and `gl_f16`, the same rows in GL texel order (row 0 = v 0 = straight down: what the sampler sees)."""
    here = os.path.dirname(os.path.abspath(__file__))
    rgbe = np.load(os.path.join(here, "assets", "spree_bank_1k_rgbe.npz"))["rgbe"]
    scale = np.exp2(rgbe[..., 3].astype(np.float64) - 128.0) / 255.0
    rgb = np.minimum(rgbe[..., :3].astype(np.float64) * scale[..., None], 65504.0)
    img = np.concatenate([rgb, np.ones_like(rgb[..., :1])], -1).astype(np.float16)
    return img, np.ascontiguousarray(img[::-1])


def load_blue_noise() -> np.ndarray:
    """128x128 RGBA8 blue-noise texture in GL texel order (flipY applied): the decoded pixels of
    the reference's src/utils/blue_noise_rgba.png (sha256 359e71ac...), made by
    tools/make_blue_noise_asset.py."""
    import os

    path = os.path.join(os.path.dirname(__file__), "assets", "blue_noise_rgba_128.bin")
    return np.fromfile(path, dtype=np.uint8).reshape(128, 128, 4)
