"""A second, independently written restatement of whole passes - vectorised numpy in float64, derived from the GLSL, sharing
no code with oracle/rfx_oracle.cpp - checked against the C++ oracle on the frames of the chain harness.

The reference ships nothing to pin the oracle to (SURVEY.md §4/§8c: parity unpinned).  Two restatements written at different
times, in different languages and styles (scalar C++ with fp32 lowering rules vs whole-image numpy in fp64) agreeing to the
fp16 quantisation of the targets is the strongest check this environment allows that the oracle follows the shader text and
not a transcription slip.  Covered: K1 SSGI trace (ssgi.frag:105-503 + ssgi_utils.frag: view position, TBN, VNDF sample,
diffuse/specular lottery, both BRDFs and pdfs, the ray march with binary refinement, hit shading with saturation and border
fade, ray length, packTwoVec4; with and without the environment map - inverse-CDF importance sample with its implicit-LOD
colour fetch, MIS weights, equirect lookup with the roughness-scaled mip and the luminance cap), K2 temporal reprojection in its SSGI form
(temporal_reproject.frag:42-208 + reproject.frag: both reprojection modes, the confidence checks, Catmull-Rom history fetch,
neighbourhood clamp, accumulation), K3 Poisson denoise (poisson_denoise.frag:52-208, both the NEAREST fp32 first pass and the
LINEAR fp16 later passes, two planes, G-buffer variant), the G-buffer material decode it uses (gbuffer_packing.glsl:24-63,
151-196), the blue-noise lookup (blue_noise.glsl:9-48), K4 GI compose (DenoiserComposePass.js:58-85 +
denoiser_compose_functions.glsl:13-107), K5 ssgi_compose.frag:20-44, K6 HBAO (hbao.frag:21-96 + hbao_utils.glsl), K7
ao_compose.frag:6-16, K8 motion blur (motion_blur.frag:11-44, incl. the tiled frame-0 lookup and a window size that differs
from the buffer size) and K9 traa_compose.frag:3-6; K1 also in MODE_SSR and K2 also in the one-plane form TRAAEffect drives.

What the exercise found: the two restatements disagreed twice, both times on a documented reference quirk that only one of
them had modelled - GLSL's fp32 `mod` on packed values above 2^24 (metalness = 1) and `max(EPSILON, NaN)` returning EPSILON -
and never on the algorithm.
"""
import warnings

import numpy as np

warnings.filterwarnings("ignore", message="invalid value encountered", category=RuntimeWarning)

import chain_harness as ch
import orc
from realism_effects_b200 import abi


# ---- leaf restatements -----------------------------------------------------------------------------------------------------
def np_unpack_half2x16(bits_f32):
    u = bits_f32.view(np.uint32)
    lo = (u & 0xFFFF).astype(np.uint16).view(np.float16).astype(np.float64)
    hi = (u >> 16).astype(np.uint16).view(np.float16).astype(np.float64)
    return lo, hi


def np_unpack_normal(packed_f32):
    """unpackNormal = decodeOctWrap(unpackHalf2x16(bits))  gbuffer_packing.glsl:52-63"""
    fx, fy = np_unpack_half2x16(packed_f32)
    fx, fy = fx * 2.0 - 1.0, fy * 2.0 - 1.0
    nz = 1.0 - np.abs(fx) - np.abs(fy)
    t = np.maximum(-nz, 0.0)
    nx = fx + np.where(fx >= 0.0, -t, t)
    ny = fy + np.where(fy >= 0.0, -t, t)
    n = np.stack([nx, ny, nz], -1)
    return n / np.linalg.norm(n, axis=-1, keepdims=True)


def np_roughness(b_f32):
    """float2color(value).r - NON_ZERO_OFFSET, clamped at 0   gbuffer_packing.glsl:24-34"""
    # GLSL mod(x, y) = x - y * floor(x / y) evaluated in fp32: with metalness = 1 the packed value exceeds 2^24 and the fp32
    # product y * floor(x / y) rounds, so the shader's result is NOT the mathematical remainder (a reference quirk, kept)
    v = b_f32.astype(np.float32)
    y = np.float32(257.0)
    r = v - y * np.floor(v / y)
    return np.maximum(r.astype(np.float64) / 256.0 - 1e-4, 0.0)


def np_pcg4d_shift(index: int, size: int = 128):
    """(pcg4d(seed(index)).xy % 0x0fffffff) % size  blue_noise.glsl:12-35, uint32 wraparound done with Python ints"""
    M = 0xFFFFFFFF
    i32 = lambda v: v & M  # noqa: E731   (int -> uvec4 conversion wraps)
    v = [i32(index), i32(index * 15843), i32(index * 31 + 4566), i32(index * 2345 + 58585)]
    v = [(x * 1664525 + 1013904223) & M for x in v]

    def rounds(v):
        v[0] = (v[0] + v[1] * v[3]) & M
        v[1] = (v[1] + v[2] * v[0]) & M
        v[2] = (v[2] + v[0] * v[1]) & M
        v[3] = (v[3] + v[1] * v[2]) & M
        return v

    v = rounds(v)
    v = [x ^ (x >> 16) for x in v]
    v = rounds(v)
    return (v[0] % 0x0FFFFFFF), (v[1] % 0x0FFFFFFF)


def np_blue_noise(blue_rgba8, index, W, H):
    sx, sy = np_pcg4d_shift(index)
    ys, xs = np.mgrid[0:H, 0:W]
    return blue_rgba8[(ys + sy) % 128, (xs + sx) % 128].astype(np.float64) / 255.0


def np_fwidth(a):
    """fine 2x2-quad derivatives: |right - left| + |lower - upper| of the pixel's quad (even image sizes)"""
    H, W = a.shape[:2]
    q = a.reshape(H // 2, 2, W // 2, 2, *a.shape[2:])
    dx = np.abs(q[:, :, :, 1] - q[:, :, :, 0])[:, :, :, None]
    dy = np.abs(q[:, 1] - q[:, 0])[:, None]
    return (np.broadcast_to(dx, q.shape) + np.broadcast_to(dy, q.shape)).reshape(a.shape)


def np_nearest(plane, u, v):
    H, W = plane.shape[:2]
    ix = np.clip(np.floor(u * W).astype(np.int64), 0, W - 1)
    iy = np.clip(np.floor(v * H).astype(np.int64), 0, H - 1)
    return plane[iy, ix]


def np_bilinear(plane, u, v):
    H, W = plane.shape[:2]
    fx, fy = u * W - 0.5, v * H - 0.5
    x0, y0 = np.floor(fx), np.floor(fy)
    ax, ay = (fx - x0)[..., None], (fy - y0)[..., None]
    cx = lambda x: np.clip(x.astype(np.int64), 0, W - 1)  # noqa: E731
    cy = lambda y: np.clip(y.astype(np.int64), 0, H - 1)  # noqa: E731
    p = plane.astype(np.float64)
    return ((p[cy(y0), cx(x0)] * (1 - ax) + p[cy(y0), cx(x0 + 1)] * ax) * (1 - ay) +
            (p[cy(y0 + 1), cx(x0)] * (1 - ax) + p[cy(y0 + 1), cx(x0 + 1)] * ax) * ay)


# ---- K3 --------------------------------------------------------------------------------------------------------------------
def np_poisson(p: abi.PoissonParams, depth, gbuffer, in0, in1, blue, prev0, prev1):
    H, W = depth.shape
    ys, xs = np.mgrid[0:H, 0:W]
    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    d = depth.astype(np.float64)
    discard = (depth == 1.0) & (np_fwidth(d) == 0.0)
    fetch = np_bilinear if p.input_linear else (lambda pl, uu, vv: np_nearest(pl, uu, vv).astype(np.float64))
    lum = lambda c: np.power(np.maximum(c @ np.array([0.2125, 0.7154, 0.0721]), 0.0), 0.125)  # noqa: E731
    planes = [in0, in1]
    rgb, alpha, lumc, age, tw = [], [], [], [], []
    for i in range(2):
        t = fetch(planes[i], u, v)
        alpha.append(t[..., 3])
        age.append(1.0 / np.power(t[..., 3] + 1.0, 1.2 * p.phi))
        c = np.log(t[..., :3] * 1.0003 + 1.0)
        rgb.append(c.copy())
        lumc.append(lum(c))
        tw.append(np.ones((H, W)))
    normal = np_unpack_normal(gbuffer[..., 1])
    rough = np_roughness(gbuffer[..., 2])
    gloss = np.maximum(0.0, 4.0 * (1.0 - rough / 0.25))
    spec_factor = np.exp(-gloss * p.specular_phi)
    flat = 1.0 - np.minimum(np.linalg.norm(np_fwidth(normal), axis=-1), 1.0)
    flat = flat ** 2 * 0.75 + 0.25
    bn = np_blue_noise(blue, p.blue_noise_index, W, H)
    ang = bn[..., 0] * 2.0 * np.pi
    s, c = np.sin(ang), np.cos(ang)
    k = p.radius * flat
    S2 = 1.41421356237
    POISSON = [(-1, 0), (0, -1), (1, 0), (0, 1), (-.25 * S2, -.25 * S2), (.25 * S2, -.25 * S2), (.25 * S2, .25 * S2), (-.25 * S2, .25 * S2)]
    for ox, oy in POISSON:
        ox, oy = ox / W, oy / H
        nu, nv = u + k * (c * ox + s * oy), v + k * (-s * ox + c * oy)   # mat2(c, -s, s, c) is column-major
        nd = np_nearest(depth, nu, nv).astype(np.float64)
        ng = np_nearest(gbuffer, nu, nv)
        nn, nr = np_unpack_normal(ng[..., 1]), np_roughness(ng[..., 2])
        ndiff = 1.0 - np.maximum((normal * nn).sum(-1), 0.0)
        w_basic = np.exp(-ndiff * p.normal_phi - 10000.0 * np.abs(d - nd) * p.depth_phi - np.abs(rough - nr) * p.roughness_phi)
        w_basic = np.where(nd == 1.0, 0.0, w_basic)
        for i in range(2):
            w = w_basic * (spec_factor if p.is_texture_specular[i] else 1.0)
            t = np.log(fetch(planes[i], nu, nv)[..., :3] + 1.0)
            disoccl = np.power(w, 0.1)
            ldiff = np.minimum(np.abs(lumc[i] - lum(t)), 0.5)
            w = (w * np.exp(-ldiff * p.luma_phi) * (1 - age[i]) + disoccl * age[i]) * age[i]
            w = np.where(w >= 0.0001, w, 0.0)
            rgb[i] += w[..., None] * t
            tw[i] += w
    outs = []
    for i, prev in enumerate((prev0, prev1)):
        o = np.concatenate([np.exp(rgb[i] / tw[i][..., None]) - 1.0, alpha[i][..., None]], -1)
        outs.append(np.where(discard[..., None], prev.astype(np.float64), o))
    return outs


def _agree(want, got, rtol, atol, max_bad):
    want, got = want.astype(np.float64), got.astype(np.float64)
    bad = np.abs(want - got) > rtol * np.maximum(np.abs(want), np.abs(got)) + atol
    frac = bad.any(-1).mean() if bad.ndim == 3 else bad.mean()
    assert frac <= max_bad, f"{frac:.2e} of the pixels differ (limit {max_bad:.0e}); worst abs {np.abs(want - got).max():.3e}"
    return frac


def test_poisson_pass_oracle_matches_numpy_restatement():
    o = ch.Opts(denoise_iterations=1, steps=8, refine_steps=2)
    inp = ch.make_inputs(96, 64, 2)
    rec = ch.run_oracle_chain(inp, o)[1]
    fr = inp.frames[1]
    seen_modes = set()
    for k3 in rec["_k3"]:
        p = k3["params"]
        seen_modes.add(int(p.input_linear))
        w0, w1 = np_poisson(p, fr["depth"], fr["gbuffer"], k3["in0"], k3["in1"], inp.blue, k3["prev0"], k3["prev1"])
        # the oracle's targets are fp16 (2^-11 relative); its arithmetic is fp32 with fixed lowering, the restatement's fp64:
        # branch flips (w >= 1e-4, nearest-texel choice on an exact half) may differ for a handful of pixels
        _agree(w0, k3["out0"], 2e-3, 1e-4, 5e-3)
        _agree(w1, k3["out1"], 2e-3, 1e-4, 5e-3)
        assert np.isfinite(w0).all() and (k3["out0"].astype(np.float64) != k3["prev0"].astype(np.float64)).any()
    assert seen_modes == {0, 1}  # the NEAREST fp32 first pass and a LINEAR fp16 pass were both exercised


def test_material_decode_matches_oracle_unpack():
    import ctypes as C

    L = orc.lib()
    inp = ch.make_inputs(64, 32, 1)
    g = inp.frames[0]["gbuffer"].reshape(-1, 4)
    geo = inp.frames[0]["depth"].reshape(-1) < 1.0
    n_np, r_np = np_unpack_normal(g[:, 1].copy()), np_roughness(g[:, 2].copy())
    out = np.zeros(12, np.float32)
    for i in np.flatnonzero(geo)[::7]:
        tex = np.ascontiguousarray(g[i])
        L.orc_unpack_gbuffer(tex.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))  # diffuse4, normal3, roughness, metalness, emissive3
        assert np.allclose(out[4:7], n_np[i], atol=2e-6) and abs(out[7] - r_np[i]) < 2e-6


def test_blue_noise_shift_matches_oracle():
    import ctypes as C

    L = orc.lib()
    for index in (1, 2, 77, 991, 123456, 2 ** 31 - 2):
        sx, sy = np_pcg4d_shift(index)
        ox, oy = C.c_int(), C.c_int()
        L.orc_blue_noise_coord(5, 9, index, 128, C.byref(ox), C.byref(oy))
        assert (ox.value, oy.value) == ((5 + sx) % 128, (9 + sy) % 128)


def test_ao_and_traa_compose_match_numpy_restatement():
    rng = np.random.default_rng(3)
    H, W = 24, 40
    depth = rng.random((H, W)).astype(np.float32)
    depth[rng.random((H, W)) < 0.2] = 1.0
    ao = rng.random((H, W, 4)).astype(np.float16)
    col = (rng.random((H, W, 4)) * 3).astype(np.float16)
    # ao_compose.frag:6-16: mix(color, 1, pow(depth > .9999 ? 1 : ao, power)) * input
    got = orc.ao_compose(ch.ao_compose_params(power=2.0, color=(0.1, 0.2, 0.3)), depth, ao, col).astype(np.float64)
    a = np.where(depth > 0.9999, 1.0, ao[..., 3].astype(np.float64)) ** 2.0
    want_rgb = (np.array([0.1, 0.2, 0.3])[None, None] * (1 - a[..., None]) + a[..., None]) * col[..., :3].astype(np.float64)
    _agree(want_rgb, got[..., :3], 2e-3, 1e-4, 0.0)
    acc = (rng.random((H, W, 4)) * 2).astype(np.float16)  # traa_compose.frag:3-6 copies the accumulated colour with alpha 1
    got = orc.traa_compose(acc).astype(np.float64)
    _agree(acc[..., :3].astype(np.float64), got[..., :3], 1e-3, 1e-6, 0.0)


# ---- K4 --------------------------------------------------------------------------------------------------------------------
def np_float_to_vec4(f32):
    """floatToVec4  gbuffer_packing.glsl:151-164: bytes / 255 - 1e-4, clamped at 0"""
    u = f32.view(np.uint32)
    v = np.stack([(u >> s) & 0xFF for s in (0, 8, 16, 24)], -1).astype(np.float64) / 255.0
    return np.maximum(v - 1e-4, 0.0)


def np_metalness(b_f32):
    v = b_f32.astype(np.float32)  # fp32 like the shader (see np_roughness)
    return np.maximum(np.floor(v / np.float32(257.0 * 257.0)).astype(np.float64) / 256.0 - 1e-4, 0.0)


def np_normalize(a):
    return a / np.linalg.norm(a, axis=-1, keepdims=True)


def np_gi_compose(cam: dict, depth, gbuffer, dgi, sgi, prev, flips: list | None = None):
    """DenoiserComposePass.js:58-85 + constructGlobalIllumination (denoiser_compose_functions.glsl:53-107), inputType DIFFUSE_SPECULAR.
    cam: synth camera uniforms (column-major 4x4 arrays).  flips: if a list, the mask of the composed pixels that take the
    `dot(viewNormal, l) < 0` flip is appended to it."""
    H, W = depth.shape
    M = lambda k: np.asarray(cam[k], np.float64).reshape(4, 4).T  # noqa: E731  column-major -> numpy row-major
    P, Pinv, Mw, V = M("projection"), M("projection_inverse"), M("camera_matrix_world"), M("view_matrix")
    near, far = float(cam["near"]), float(cam["far"])
    ys, xs = np.mgrid[0:H, 0:W]
    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    d = depth.astype(np.float64)
    discard = (depth == 1.0) & (np_fwidth(d) == 0.0)
    diffuse = np_float_to_vec4(gbuffer[..., 0].copy())[..., :3]
    normal = np_unpack_normal(gbuffer[..., 1].copy())
    rough, metal = np_roughness(gbuffer[..., 2]), np_metalness(gbuffer[..., 2])
    rgbe = np_float_to_vec4(gbuffer[..., 3].copy())
    emissive = rgbe[..., :3] * np.exp2(rgbe[..., 3:4] * 255.0 - 128.0)
    rot_left = lambda vec, A: vec @ A[:3, :3]          # noqa: E731  (vec4(v, 0) * A).xyz = A^T v, i.e. row-vector times A
    view_normal = rot_left(normal, Mw)
    view_z = -(near * far / ((far - near) * d - far))   # -perspectiveDepthToViewZ
    clip_w = P[3, 2] * view_z + P[3, 3]                 # projectionMatrix[2][3] is column 2, row 3
    clip = np.stack([(u - 0.5) * 2.0, (v - 0.5) * 2.0, (view_z - 0.5) * 2.0, np.ones_like(u)], -1) * clip_w[..., None]
    pos = clip @ Pinv.T
    view_pos = np.stack([pos[..., 0], pos[..., 1], -view_z], -1)
    view_dir = np_normalize(view_pos)
    a = (rough * rough)[..., None]
    N = rot_left(view_normal, V)
    vv = -view_dir
    Vw = rot_left(vv, V)
    up = np.where((np.abs(N[..., 2:3]) < 0.9999999), np.array([0.0, 0.0, 1.0]), np.array([1.0, 0.0, 0.0]))
    T = np_normalize(np.cross(up, N))
    B = np.cross(N, T)
    Vl = np.stack([(Vw * T).sum(-1), (Vw * B).sum(-1), (Vw * N).sum(-1)], -1)
    # SampleGGXVNDF(V, a, a, 0.25, 0.25)
    Vh = np_normalize(np.concatenate([a * Vl[..., :2], Vl[..., 2:3]], -1))
    lensq = Vh[..., 0] ** 2 + Vh[..., 1] ** 2
    T1 = np.where((lensq > 0.0)[..., None], np.stack([-Vh[..., 1], Vh[..., 0], np.zeros_like(lensq)], -1) / np.sqrt(np.maximum(lensq, 1e-300))[..., None],
                  np.array([1.0, 0.0, 0.0]))
    T2 = np.cross(Vh, T1)
    r, phi = np.sqrt(0.25), 2.0 * np.pi * 0.25
    t1, t2 = r * np.cos(phi), r * np.sin(phi)
    s = 0.5 * (1.0 + Vh[..., 2])
    t2 = (1.0 - s) * np.sqrt(1.0 - t1 * t1) + s * t2
    Nh = t1 * T1 + t2[..., None] * T2 + np.sqrt(np.maximum(0.0, 1.0 - t1 * t1 - t2 * t2))[..., None] * Vh
    Hh = np_normalize(np.concatenate([a * Nh[..., :2], np.maximum(0.0, Nh[..., 2:3])], -1))
    Hh = np.where(Hh[..., 2:3] < 0.0, -Hh, Hh)
    inc = -Vl
    l = np_normalize(inc - 2.0 * (Hh * inc).sum(-1, keepdims=True) * Hh)   # reflect(-V, H)
    l = l[..., 0:1] * T + l[..., 1:2] * B + l[..., 2:3] * N
    l = np_normalize(rot_left(l, Mw))  # (vec4(l, 1.) * cameraMatrixWorld).xyz: the translation row only feeds .w
    flip = (view_normal * l).sum(-1) < 0.0
    if flips is not None:
        flips.append(flip & ~discard)
    l = np.where(flip[..., None], -l, l)
    h = np_normalize(vv + l)
    # GLSL max(x, y) = (x < y) ? y : x.  With roughness 0 on a back-facing texel H = normalize(0) is NaN, the comparison with
    # NaN is false and max(EPSILON, NaN) returns EPSILON - the shader's output there is finite (F ~ 1), and so is the oracle's.
    dvh = (vv * h).sum(-1)
    VoH = np.where(1e-6 < dvh, dvh, 1e-6)[..., None]
    f0 = 0.04 * (1.0 - metal[..., None]) + diffuse * metal[..., None]
    F = f0 + (1.0 - f0) * np.power(1.0 - VoH, 5.0)
    gi = diffuse * (1.0 - metal[..., None]) * (1.0 - F) * dgi[..., :3].astype(np.float64) + sgi[..., :3].astype(np.float64) * F + emissive
    out = np.concatenate([gi, np.ones((H, W, 1))], -1)
    return np.where(discard[..., None], prev.astype(np.float64), out)


def test_gi_compose_oracle_matches_numpy_restatement():
    o = ch.Opts(denoise_iterations=1, steps=8, refine_steps=2)
    inp = ch.make_inputs(96, 64, 2)
    recs = ch.run_oracle_chain(inp, o)
    for t in (0, 1):
        fr, rec = inp.frames[t], recs[t]
        want = np_gi_compose(fr["cam"], fr["depth"], fr["gbuffer"], rec["dn0"], rec["dn1"], rec["_k4_prev"])
        frac = _agree(want, rec["composed"], 1e-3, 1e-5, 0.0)    # fp32 oracle vs fp64 restatement, through pow(1 - VoH, 5)
        assert _agree(want, rec["composed"], 3e-4, 1e-5, 3e-3) < 3e-3 and np.isfinite(want).all() and frac == 0.0


# ---- K1 (no environment map, no importance sampling: the ray march, the lottery, the BRDFs and the hit shading) ------------
EPS = 0.00001


def _dot(a, b):
    return (a * b).sum(-1)


def _clamp_angle(x):
    return np.clip(x, EPS, 1.0 - EPS)


def np_sample_ggx_vndf(V, a, r1, r2):
    """SampleGGXVNDF(V, a, a, r1, r2)  ssgi_utils.frag:153-170"""
    a = a[..., None]
    Vh = np_normalize(np.concatenate([a * V[..., :2], V[..., 2:3]], -1))
    lensq = Vh[..., 0] ** 2 + Vh[..., 1] ** 2
    T1 = np.where((lensq > 0.0)[..., None], np.stack([-Vh[..., 1], Vh[..., 0], np.zeros_like(lensq)], -1) / np.sqrt(np.maximum(lensq, 1e-300))[..., None],
                  np.array([1.0, 0.0, 0.0]))
    T2 = np.cross(Vh, T1)
    r, phi = np.sqrt(r1), 2.0 * np.pi * r2
    t1, t2 = r * np.cos(phi), r * np.sin(phi)
    s = 0.5 * (1.0 + Vh[..., 2])
    t2 = (1.0 - s) * np.sqrt(1.0 - t1 * t1) + s * t2
    Nh = t1[..., None] * T1 + t2[..., None] * T2 + np.sqrt(np.maximum(0.0, 1.0 - t1 * t1 - t2 * t2))[..., None] * Vh
    return np_normalize(np.concatenate([a * Nh[..., :2], np.maximum(0.0, Nh[..., 2:3])], -1))


def np_env_mips(env_f16):
    """box-filtered mip chain of a power-of-two equirect map, every level rounded to fp16 (GL generateMipmap, SURVEY.md A4)"""
    levels = [env_f16.astype(np.float64)]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        a = levels[-1]
        h, w = a.shape[:2]
        y0, y1 = np.minimum(2 * np.arange(max(1, h // 2)), h - 1), np.minimum(2 * np.arange(max(1, h // 2)) + 1, h - 1)
        x0, x1 = np.minimum(2 * np.arange(max(1, w // 2)), w - 1), np.minimum(2 * np.arange(max(1, w // 2)) + 1, w - 1)
        b = (a[y0][:, x0] + a[y0][:, x1] + a[y1][:, x0] + a[y1][:, x1]) * 0.25
        levels.append(b.astype(np.float16).astype(np.float64))
    return levels


def np_trilinear(mips, eu, ev, lod):
    """textureLod(map, uv, lod), LINEAR_MIPMAP_LINEAR, clamp to edge"""
    n = len(mips)
    l = np.clip(lod, 0.0, n - 1.0)
    l0 = np.floor(l).astype(np.int64)
    l1 = np.minimum(l0 + 1, n - 1)
    f = (l - l0)[..., None]
    A, B = np.zeros(eu.shape + (4,)), np.zeros(eu.shape + (4,))
    for k in range(n):
        if (l0 == k).any() or (l1 == k).any():
            s = np_bilinear(mips[k], eu, ev)
            A, B = np.where((l0 == k)[..., None], s, A), np.where((l1 == k)[..., None], s, B)
    return A * (1.0 - f) + B * f


def np_equirect_uv(dirs):
    """equirectDirectionToUv  ssgi_utils.frag:64-74"""
    return np.arctan2(dirs[..., 2], dirs[..., 0]) / (2.0 * np.pi) + 0.5, 1.0 - np.arccos(np.clip(dirs[..., 1], -1.0, 1.0)) / np.pi


def np_ssgi_trace(p: abi.SsgiParams, depth, gbuffer, direct, accumulated, blue, env=None):
    """ssgi.frag:105-503 + ssgi_utils.frag, MODE_SSGI, missedRays undefined, with or without USE_ENVMAP + importanceSampling (env =
    (map fp16 (h, w, 4), marginal, conditional, total_sum)); the velocity sampler is the null sampler of the shipped wiring
    (SURVEY.md D4).  Returns the 8 stored fp16 channels as float64."""
    use_env, use_is = bool(p.flags & abi.SSGI_USE_ENVMAP), bool(p.flags & abi.SSGI_IMPORTANCE_SAMPLING)
    assert not (p.flags & abi.SSGI_MISSED_RAYS) and (env is not None or not (use_env or use_is))
    ssr = p.mode == abi.MODE_SSR
    H, W = depth.shape
    cam = p.cam
    M = lambda arr: np.asarray(list(arr), np.float64).reshape(4, 4).T  # noqa: E731
    P, Pinv, Mw, V_ = M(cam.projection), M(cam.projection_inverse), M(cam.camera_matrix_world), M(cam.view_matrix)
    near, far = float(cam.near_plane), float(cam.far_plane)
    rot_left = lambda vec, A: vec @ A[:3, :3]  # noqa: E731
    ys, xs = np.mgrid[0:H, 0:W]
    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    d = depth.astype(np.float64)
    view_z_of = lambda dd: (near * far) / ((far - near) * dd - far)  # noqa: E731
    project = lambda pos: tuple(((np.concatenate([pos, np.ones_like(pos[..., :1])], -1) @ P.T)[..., k] /  # noqa: E731
                                 (np.concatenate([pos, np.ones_like(pos[..., :1])], -1) @ P.T)[..., 3]) * 0.5 + 0.5 for k in (0, 1))
    lum = lambda c: c @ np.array([0.2125, 0.7154, 0.0721])  # noqa: E731

    diffuse = np_float_to_vec4(gbuffer[..., 0].copy())[..., :3]
    normal = np_unpack_normal(gbuffer[..., 1].copy())
    rough, metal = np_roughness(gbuffer[..., 2]), np_metalness(gbuffer[..., 2])
    rsq = np.clip(rough * rough, 0.000001, 1.0)
    view_z = view_z_of(d)
    clip_w = P[3, 2] * view_z + P[3, 3]
    clip = np.stack([(u - 0.5) * 2.0, (v - 0.5) * 2.0, (view_z - 0.5) * 2.0, np.ones_like(u)], -1) * clip_w[..., None]
    vp = clip @ Pinv.T
    view_pos = np.stack([vp[..., 0], vp[..., 1], view_z], -1)
    view_dir = np_normalize(view_pos)
    view_normal = np_normalize(rot_left(normal, Mw))
    n, vv = view_normal, -view_dir
    NoV = np.where(EPS < _dot(n, vv), _dot(n, vv), EPS)
    Vw = rot_left(vv, V_)
    N = normal
    up = np.where((np.abs(N[..., 2:3]) < 0.9999999), np.array([0.0, 0.0, 1.0]), np.array([1.0, 0.0, 0.0]))
    T = np_normalize(np.cross(up, N))
    B = np.cross(N, T)
    Vl = np.stack([_dot(Vw, T), _dot(Vw, B), _dot(Vw, N)], -1)
    f0 = 0.04 * (1.0 - metal[..., None]) + diffuse * metal[..., None]
    rnd = np_blue_noise(blue, p.blue_noise_index, W, H)
    Hh = np_sample_ggx_vndf(Vl, rsq, rnd[..., 0], rnd[..., 1])
    Hh = np.where(Hh[..., 2:3] < 0.0, -Hh, Hh)
    inc = -Vl
    l = np_normalize(inc - 2.0 * _dot(Hh, inc)[..., None] * Hh)
    l = l[..., 0:1] * T + l[..., 1:2] * B + l[..., 2:3] * N
    l = np_normalize(rot_left(l, Mw))

    def angles(ll):
        h = np_normalize(vv + ll)
        return _clamp_angle(_dot(n, ll)), _clamp_angle(_dot(n, h)), _clamp_angle(_dot(ll, h)), _clamp_angle(_dot(vv, h))

    _, _, _, VoH = angles(l)
    F = f0 + (1.0 - f0) * np.power(1.0 - VoH, 5.0)[..., None]
    diffW = np.maximum((1.0 - metal) * lum(diffuse), EPS)
    specW = np.maximum(lum(F), EPS)
    diffW = diffW * (1.0 / (diffW + specW))
    is_diffuse = (rnd[..., 2] < diffW) & (not ssr)   # MODE_SSR never takes a diffuse sample (:188-190)
    # cosineSampleHemisphere(viewNormal, random.rg)  ssgi_utils.frag:183-191
    r_, th = np.sqrt(rnd[..., 0]), 2.0 * np.pi * rnd[..., 1]
    b_ = np_normalize(np.cross(n, np.broadcast_to(np.array([0.0, 1.0, 1.0]), n.shape)))
    t_ = np.cross(b_, n)
    diffuse_ray = np_normalize((r_ * np.sin(th))[..., None] * b_ + np.sqrt(1.0 - rnd[..., 0])[..., None] * n + (r_ * np.cos(th))[..., None] * t_)
    spec_ray = l
    ems_pdf, is_env = np.ones((H, W)), np.zeros((H, W), bool)
    if use_env or use_is:
        mips = np_env_mips(env[0])
        eh, ew = env[0].shape[:2]
    if use_is:  # sampleEquirectProbability  ssgi_utils.frag:210-225 and ssgi.frag:197-215
        marg, cond = np.asarray(env[1], np.float64), np.asarray(env[2], np.float64)
        cv = marg[np.clip(np.floor(rnd[..., 0] * len(marg)).astype(np.int64), 0, len(marg) - 1)]
        cu = cond[np.clip(np.floor(cv * eh).astype(np.int64), 0, eh - 1), np.clip(np.floor(rnd[..., 1] * ew).astype(np.int64), 0, ew - 1)]
        theta, phi = (cu - 0.5) * 2.0 * np.pi, (1.0 - cv) * np.pi
        edir = np.stack([np.sin(phi) * np.cos(theta), np.cos(phi), np.sin(phi) * np.sin(theta)], -1)
        # texture(info.map, uv): implicit LOD from the quad derivatives of the (random) uv, in texels
        q = np.stack([cu * ew, cv * eh], -1).reshape(H // 2, 2, W // 2, 2, 2)
        ddx = np.linalg.norm(q[:, :, :, 1] - q[:, :, :, 0], axis=-1)[:, :, :, None]
        ddy = np.linalg.norm(q[:, 1] - q[:, 0], axis=-1)[:, None]
        rho = np.maximum(np.broadcast_to(ddx, (H // 2, 2, W // 2, 2)), np.broadcast_to(ddy, (H // 2, 2, W // 2, 2))).reshape(H, W)
        lam = np.where(rho > 0.0, np.log2(np.maximum(rho, 1e-300)), -1000.0)
        ecol = np_trilinear(mips, cu, cv, lam)[..., :3]
        ems_pdf = ew * eh * lum(ecol) / float(env[3])
        edir = np_normalize(rot_left(edir, Mw))
        prob = np.minimum(1.0 - EPS, _dot(edir, view_normal) * rough)
        is_env = rnd[..., 3] < prob
        ems_pdf = np.where(is_env, ems_pdf / (1.0 - prob), 1.0 - prob)
        diffuse_ray = np.where(is_env[..., None], edir, diffuse_ray)
        spec_ray = np.where(is_env[..., None], edir, spec_ray)

    def env_color(ll, diffuse_sample):  # getEnvColor  ssgi.frag:311-346
        if not use_env:
            return np.zeros((H, W, 3))
        eu, ev = np_equirect_uv(np_normalize(rot_left(ll, V_)))
        mip = np.full((H, W), p.env_blur * p.max_env_map_mip_level)
        if not diffuse_sample:
            mip = np.where(rsq < 0.15, mip * (rsq / 0.15), mip)
        s = np_trilinear(mips, eu, ev, mip)[..., :3]
        cap = np.where(is_env, 100.0, 25.0)
        el = lum(s)
        return np.where((el > cap)[..., None], s * (cap / np.where(el == 0.0, 1.0, el))[..., None], s)

    def d_gtr2(a, NoH):
        a2 = a * a
        return a2 / (np.pi * ((NoH * NoH) * (a2 * a2 - 1.0) + 1.0) ** 2)

    def smith_g(NdV, alpha):
        a, b = alpha * alpha, NdV * NdV
        return (2.0 * NdV) / (NdV + np.sqrt(a + b - a * b))

    def do_sample(ll, diffuse_sample):
        NoL, NoH, LoH, _ = angles(ll)
        cos_theta = np.maximum(0.0, _dot(view_normal, ll))
        if diffuse_sample:
            fd90 = 0.5 + 2.0 * rsq * LoH * LoH
            fs = lambda th_: 1.0 + (fd90 - 1.0) * np.power(1.0 - th_, 5.0)  # noqa: E731
            brdf = (fs(NoL) * fs(NoV) / np.pi) * (1.0 - metal)
            pdf = NoL / np.pi
        else:
            ag = (0.5 + rsq * 0.5) ** 2
            G = smith_g(NoV, ag * ag) * smith_g(NoL, ag * ag)
            brdf = d_gtr2(rsq, NoH) * G / (4.0 * NoL * NoV)
            pdf = d_gtr2(rsq, NoH) * smith_g(NoV, rsq * rsq) / np.maximum(0.00001, 4.0 * NoV)
        brdf = brdf * cos_theta
        pdf = np.maximum(EPS, pdf)
        # RayMarch  ssgi.frag:441-475
        dirv = ll * (p.ray_distance / float(p.steps))
        pos = view_pos.copy()
        hit = np.zeros((H, W), bool)
        for i in range(1, p.steps):
            cs = 1.0 - np.exp(-0.25 * (i + rnd[..., 2] - 0.5) ** 2)
            pos = np.where(hit[..., None], pos, pos + dirv * cs[..., None])
            pu, pv = project(pos)
            diff = view_z_of(np_nearest(depth, pu, pv).astype(np.float64)) - pos[..., 2]
            hit = hit | ((diff >= 0.0) & (diff < p.thickness))
        if p.refine_steps > 0:  # BinarySearch :477-503 (for the rays that hit)
            dr = dirv * 0.5
            rp = pos - dr
            for _ in range(p.refine_steps):
                pu, pv = project(rp)
                diff = view_z_of(np_nearest(depth, pu, pv).astype(np.float64)) - rp[..., 2]
                dr = dr * 0.5
                rp = np.where((diff >= 0.0)[..., None], rp - dr, rp + dr)
            pos = np.where(hit[..., None], rp, pos)
        cu, cv = project(pos)
        inside = (cu >= 0.0) & (cu <= 1.0) & (cv >= 0.0) & (cv <= 1.0)
        rgi = np_nearest(accumulated, cu, cv)[..., :3].astype(np.float64)
        mx, mn = diffuse.max(-1), diffuse.min(-1)
        sat = np.where(mx == mn, 0.0, (mx - mn) / np.where(mx == 0.0, 1.0, mx))
        k = ((1.0 - rsq) * sat * 0.4)[..., None]
        rgi = rgi * (1.0 - k) + lum(rgi)[..., None] * k
        sm = lambda e0, e1, x: (lambda t: t * t * (3.0 - 2.0 * t))(np.clip((x - e0) / (e1 - e0), 0.0, 1.0))  # noqa: E731
        bf = np.sqrt(sm(0.0, 0.15, cu) * sm(1.0, 0.85, cu) * sm(0.0, 0.15, cv) * sm(1.0, 0.85, cv))[..., None]
        ec = env_color(ll, diffuse_sample)   # (the shader passes the march-scaled l; it is normalised inside, so the scale drops out)
        gi = np.where((hit & inside)[..., None], ec * (1.0 - bf) + rgi * bf, ec)   # miss or off-screen reprojection: the env colour alone
        gi = gi * brdf[..., None]
        aa, bb = ems_pdf * ems_pdf, pdf * pdf                               # misHeuristic for env samples, plain 1/pdf otherwise
        gi = np.where(is_env[..., None], gi * (aa / (aa + bb))[..., None], gi / pdf[..., None]) / ems_pdf[..., None]
        return gi, np.where(hit[..., None], pos, 10.0e9)

    gi_d, _ = do_sample(diffuse_ray, True)
    # the specular sample evaluates the diffuse BRDF when the pixel drew the diffuse lottery (isDiffuseSample is passed through :246-249)
    gi_s_spec, hit_pos = do_sample(spec_ray, False)
    gi_s_diff, _ = do_sample(spec_ray, True)
    gi_s = np.where(is_diffuse[..., None], gi_s_diff, gi_s_spec)
    dl = direct.astype(np.float64)
    if p.flags & abi.SSGI_USE_DIRECT_LIGHT:
        gi_d, gi_s = gi_d + dl[..., :3], gi_s + dl[..., :3]
    gi_d = np.where(is_diffuse[..., None], gi_d, -1.0)
    cam_pos = Mw[:3, 3]
    hp_ws = np.concatenate([hit_pos, np.ones((H, W, 1))], -1) @ Mw.T
    ray_len = np.where(hit_pos[..., 0] > 10.0e8, 0.0, np.linalg.norm(cam_pos - hp_ws[..., :3], axis=-1))
    bg = (np.concatenate([dl, dl], -1) + 1e-4).astype(np.float16)   # the background branch packs two vec4 in BOTH modes (:109-113)
    if ssr:  # MODE_SSR: plain RGBA32F texel (specularGI, bits of packHalf2x16(rayLength, roughness))  :298-308
        alpha = np.stack([ray_len, rough], -1).astype(np.float16)
        out = np.concatenate([gi_s.astype(np.float32), alpha.view(np.float32).reshape(H, W, 1)], -1)
        return np.where((depth == 1.0)[..., None], bg.view(np.float32).reshape(H, W, 4), out)
    out = np.concatenate([gi_d, rough[..., None], gi_s, ray_len[..., None]], -1)
    out = (out + 1e-4).astype(np.float16)                           # packTwoVec4: the stored fp16 values carry the +1e-4 offset
    return np.where((depth == 1.0)[..., None], bg, out).astype(np.float64)


import pytest  # noqa: E402


@pytest.mark.parametrize("env_on", [False, True])
def test_ssgi_trace_oracle_matches_numpy_restatement(env_on):
    o = ch.Opts(use_envmap=env_on, importance_sampling=env_on, use_direct_light=True, steps=10, refine_steps=3, denoise_iterations=1)
    inp = ch.make_inputs(96, 64, 2)
    recs = ch.run_oracle_chain(inp, o)
    env = (inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total) if env_on else None
    for t in (0, 1):
        fr, rec = inp.frames[t], recs[t]
        want = np_ssgi_trace(rec["_k1_params"], fr["depth"], fr["gbuffer"], fr["direct"], rec["_k1_accumulated"], inp.blue, env)
        got = ch.unpack_halves(rec["ssgi"]).astype(np.float64)
        # discrete choices (lottery vs an 8-bit noise value, hit tests, nearest texels) can flip between fp32 and fp64 for a few rays
        frac = _agree(want, got, 3e-3, 3e-4, 1.5e-2)
        geo = fr["depth"] < 1.0
        assert frac < 1.5e-2 and (want[geo][:, 0] < -0.9).any() and (want[geo][:, 0] >= 0.0).any() and (want[geo][:, 7] > 1.0).any()


def test_ssr_mode_trace_oracle_matches_numpy_restatement():
    o = ch.Opts(mode=abi.MODE_SSR, steps=10, refine_steps=3, denoise_iterations=1)
    inp = ch.make_inputs(96, 64, 2)
    recs = ch.run_oracle_chain(inp, o)
    env = (inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    for t in (0, 1):
        fr, rec = inp.frames[t], recs[t]
        want = np_ssgi_trace(rec["_k1_params"], fr["depth"], fr["gbuffer"], fr["direct"], rec["_k1_accumulated"], inp.blue, env)
        got, geo = rec["ssgi"], fr["depth"] < 1.0
        assert _agree(want[..., :3][geo].astype(np.float64), got[..., :3][geo].astype(np.float64), 1e-3, 1e-5, 1.5e-2) < 1.5e-2
        wa = np.ascontiguousarray(want[..., 3]).view(np.uint32)[geo]     # packed (rayLength, roughness) halves
        ga = np.ascontiguousarray(got[..., 3]).view(np.uint32)[geo]
        assert ((wa >> 16) == (ga >> 16)).all()                           # roughness: exact
        rl = lambda a: (a & 0xFFFF).astype(np.uint16).view(np.float16).astype(np.float64)  # noqa: E731
        assert _agree(rl(wa), rl(ga), 2e-3, 1e-3, 1.5e-2) < 1.5e-2        # ray length: to fp16, a few rays flip hit / miss
        assert (want[~geo].view(np.uint32) == got[~geo].view(np.uint32)).all()   # background texels: bit-equal packing of the direct light


# ---- K2 (SSGI form: two planes, packed K1 input, log transform, LINEAR fp16 history) -----------------------------------------
def np_temporal(p: abi.TemporalParams, ssgi_packed, velocity, hist, prev_out):
    """temporal_reproject.frag:42-208 + reproject.frag (inputType DIFFUSE_SPECULAR, textureCount 2, logTransform)."""
    traa = p.input_type == abi.INPUT_DIFFUSE   # the one-plane form TRAAEffect drives: RGBA16F composer input, no discard, no hit-point reprojection
    assert (traa and p.texture_count == 1) or (p.input_type == abi.INPUT_DIFFUSE_SPECULAR and p.texture_count == 2)
    assert p.log_transform and p.history_linear
    H, W = velocity.shape[:2]
    M = lambda arr: np.asarray(list(arr), np.float64).reshape(4, 4).T  # noqa: E731
    cam = p.cam
    Pinv, Mw = M(cam.projection_inverse), M(cam.camera_matrix_world)
    pV, pMw, pP, pPinv = M(p.prev_view_matrix), M(p.prev_camera_matrix_world), M(p.prev_projection), M(p.prev_projection_inverse)
    near, far = float(cam.near_plane), float(cam.far_plane)
    cam_pos = np.array(list(p.camera_pos), np.float64)
    ys, xs = np.mgrid[0:H, 0:W]
    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    hom = lambda a: np.concatenate([a, np.ones_like(a[..., :1])], -1)  # noqa: E731

    def to_world(uu, vv_, dd, world, proj_inv):  # screenSpaceToWorldSpace  reproject.frag:21-28
        ndc = np.stack([(uu - 0.5) * 2.0, (vv_ - 0.5) * 2.0, (dd - 0.5) * 2.0, np.ones_like(uu)], -1)
        clip = ndc @ proj_inv.T
        return ((clip / clip[..., 3:4]) @ world.T)[..., :3]

    vel = velocity[..., :2].astype(np.float64)
    wnormal = np_unpack_normal(velocity[..., 2].copy())
    depth = velocity[..., 3].astype(np.float64)
    if traa:
        halves = ssgi_packed.astype(np.float64)                                # LINEAR fetch at the pixel centre = the texel
        inp = [halves.copy()]
    else:
        halves = ch.unpack_halves(ssgi_packed).astype(np.float64) - 1e-4      # unpackTwoVec4
        inp = [halves[..., 0:4].copy(), halves[..., 4:8].copy()]
    sampled = [t[..., 0] >= 0.0 for t in inp]
    for t in inp:
        t[..., :3] = np.log(np.maximum(t[..., :3], 0.0) + 1.0)
    discard = (velocity[..., 3] == 1.0) & (np_fwidth(depth) == 0.0) & (not traa)
    curvature = np.linalg.norm(np_fwidth(wnormal), axis=-1)
    wpos = to_world(u, v, depth, Mw, Pinv)
    ray_len, rough = (np.zeros((H, W)), np.ones((H, W))) if traa else (inp[1][..., 3], np.clip(inp[0][..., 3], 0.0, 1.0))
    view_z = np.abs(near * far / ((far - near) * depth - far))
    dist_factor = 1.0 + 1.0 / (view_z + 1.0)

    def validate(ru, rv):  # validateReprojectedUV :130-167 (confidence already raised to confidencePower once here)
        outside = (ru > 1.0) | (ru < 0.0) | (rv > 1.0) | (rv < 0.0)
        t = np_nearest(velocity, ru, rv)
        ln, ld = np_unpack_normal(np.ascontiguousarray(t[..., 2])), t[..., 3].astype(np.float64)
        lpos = to_world(ru, rv, ld, pMw, pPinv)
        dpos = wpos - lpos
        dis = (np.linalg.norm(dpos, axis=-1) / 10.0 + np.abs(_dot(dpos, wnormal)) / 20.0 + np.minimum(1.0 - _dot(wnormal, ln), 1.0)) * dist_factor
        conf = np.power(np.maximum(1.0 - np.minimum(dis, 1.0), 0.0), p.confidence_power)
        return np.where(outside, 0.0, conf)

    du, dv = u - vel[..., 0], v - vel[..., 1]
    uvc_d = (du, dv, validate(du, dv))
    ray = np_normalize(wpos - cam_pos)
    hitp = hom(cam_pos + ray * ray_len[..., None]) @ (pP @ pV).T
    su, sv = hitp[..., 0] / hitp[..., 3] * 0.5 + 0.5, hitp[..., 1] / hitp[..., 3] * 0.5 + 0.5
    no_hit = (curvature > 0.05) | (ray_len < 0.01)
    su, sv = np.where(no_hit, -1.0, su), np.where(no_hit, -1.0, sv)
    sc = validate(su, sv)
    fall = su == -1.0
    uvc_s = (np.where(fall, uvc_d[0], su), np.where(fall, uvc_d[1], sv), np.where(fall, uvc_d[2], sc))
    move = np.minimum(_dot(vel, vel) * 10000.0, 1.0)

    def catmull(plane, pu, pv):  # BiCubicCatmullRom5Tap :212-255 over a LINEAR fp16 plane
        inv = np.array([1.0 / W, 1.0 / H])
        UV = np.stack([pu, pv], -1) / inv
        tc = np.floor(UV - 0.5) + 0.5
        f = UV - tc
        f2, f3 = f * f, f * f * f
        w0, w1, w3 = f2 - 0.5 * (f3 + f), 1.5 * f3 - 2.5 * f2 + 1.0, 0.5 * (f3 - f2)
        w2 = 1.0 - w0 - w1 - w3
        W0, W1, W2 = w0, w1 + w2, w3
        S0, S1, S2 = (tc - 1.0) * inv, (tc + w2 / W1) * inv, (tc + 2.0) * inv
        taps = [(S1[..., 0], S0[..., 1], W1[..., 0] * W0[..., 1]), (S0[..., 0], S1[..., 1], W0[..., 0] * W1[..., 1]), (S1[..., 0], S1[..., 1], W1[..., 0] * W1[..., 1]),
                (S2[..., 0], S1[..., 1], W2[..., 0] * W1[..., 1]), (S1[..., 0], S2[..., 1], W1[..., 0] * W2[..., 1])]
        acc = sum(np_bilinear(plane, a, b) * w[..., None] for a, b, w in taps)
        return np.maximum(acc / sum(w for _a, _b, w in taps)[..., None], 0.0)

    lin = [np.exp(t[..., :3]) - 1.0 for t in inp]  # undoColorTransform(inputColor) for the clamp box
    outs = []
    for i in range(p.texture_count):
        spec = bool(p.reproject_specular[i])
        uvc = uvc_s if spec else uvc_d
        acc = catmull(hist[i], uvc[0], uvc[1])
        acc_rgb, acc_a = np.log(acc[..., :3] + 1.0), acc[..., 3] + 1.0
        radius = np.where(spec & (rough < 0.25), 1, 2)
        mn, mx = lin[i].copy(), lin[i].copy()
        for dy in range(-2, 3):
            for dx in range(-2, 3):
                t = halves[np.clip(ys + dy, 0, H - 1), np.clip(xs + dx, 0, W - 1)][..., 4 * i:4 * i + 3]
                use = ((np.abs(dx) <= radius) & (np.abs(dy) <= radius) & (t[..., 0] >= 0.0))[..., None]
                mn, mx = np.where(use, np.minimum(t, mn), mn), np.where(use, np.maximum(t, mx), mx)
        clamped = np.clip(acc_rgb, np.log(mn + 1.0), np.log(mx + 1.0))
        r = rough if spec else 1.0
        intensity = np.minimum(1.0, move * 50.0 + p.neighborhood_clamp_intensity) * np.minimum(1.0, uvc[2] * r)
        new = acc_rgb * (1.0 - intensity[..., None]) + clamped * intensity[..., None]
        acc_a2 = acc_a * (1.0 - np.minimum(np.linalg.norm(new - acc_rgb, axis=-1), 1.0))
        # not sampled this frame: the input is replaced by the history and the history is used as fetched (no clamp, no age + 1)
        in_rgb = np.where(sampled[i][..., None], inp[i][..., :3], acc_rgb)
        acc_rgb = np.where(sampled[i][..., None], new, acc_rgb)
        acc_a = np.where(sampled[i], acc_a2, acc[..., 3])
        conf = np.power(uvc[2], p.confidence_power)          # raised a second time in accumulate() :49
        blend = (1.0 - 1.0 / (acc_a + 1.0)) * conf
        max_v = np.full((H, W), (1.0 if p.full_accumulate else p.max_blend) * p.keep_data)
        if spec:
            low = (rough >= 0.0) & (rough < 0.1)
            mrv = max_v * (rough / 0.1)
            k = np.minimum(100.0 * move, 1.0)
            max_v = np.where(low, max_v * (1.0 - k) + mrv * k, max_v)
        tmix = np.minimum(blend, max_v)
        oa = np.minimum(65536.0, 1.0 / (1.0 - tmix) - 1.0)
        rgb = np.exp(in_rgb * (1.0 - tmix[..., None]) + acc_rgb * tmix[..., None]) - 1.0
        o = np.concatenate([rgb, oa[..., None]], -1)
        outs.append(np.where(discard[..., None], prev_out[i].astype(np.float64), o))
    return outs


def test_temporal_reproject_oracle_matches_numpy_restatement():
    o = ch.Opts(denoise_iterations=1, steps=8, refine_steps=2)
    inp = ch.make_inputs(96, 64, 3)
    recs = ch.run_oracle_chain(inp, o)
    for t in (1, 2):  # frames with a history and a moving camera
        fr, rec = inp.frames[t], recs[t]
        w0, w1 = np_temporal(rec["_k2_params"], rec["ssgi"], fr["velocity"], rec["_k2_hist"], rec["_k2_prev_out"])
        # fp32 targets; confidence / clamp branches and nearest-texel choices may flip for a few pixels between fp32 and fp64
        assert _agree(w0, rec["tr0"], 2e-4, 1e-5, 2e-3) < 2e-3   # (measured: 0 pixels outside 1e-4)
        assert _agree(w1, rec["tr1"], 2e-4, 1e-5, 2e-3) < 2e-3
        assert (rec["tr0"][..., 3] > 0.5).any()  # some history was actually accumulated


# ---- K8 motion blur, K5 ssgi compose -----------------------------------------------------------------------------------------
def np_motion_blur(p: abi.MotionBlurParams, velocity, inp_f16, blue):
    """motion_blur.frag:11-44; blueNoise(vUv, frame) with pixel = ivec2(vUv * resolution) where `resolution` is the WINDOW size"""
    H, W = velocity.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W]
    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    vel = velocity[..., :2].astype(np.float64)
    moved = _dot(vel, vel) > 0.000000001
    vel = vel * p.intensity
    rx, ry = float(p.resolution[0]), float(p.resolution[1])
    if p.frame == 0:   # tiled lookup: textureLod(blueNoise, uv * resolution / blueNoiseSize), NEAREST + REPEAT
        bx, by = np.floor(u * rx / 128.0 * 128.0).astype(np.int64) % 128, np.floor(v * ry / 128.0 * 128.0).astype(np.int64) % 128
    else:
        sx, sy = np_pcg4d_shift(p.frame)
        bx, by = (np.floor(u * rx).astype(np.int64) + sx) % 128, (np.floor(v * ry).astype(np.int64) + sy) % 128
    bn = blue[by, bx].astype(np.float64) / 255.0
    jit = p.jitter * vel * bn[..., :2]
    speed = (1.0 / 100.0) / p.delta_time
    start = np.maximum(0.0, np.stack([u, v], -1) + (jit - vel * 0.5) * speed)
    end = np.minimum(1.0, np.stack([u, v], -1) + (jit + vel * 0.5) * speed)
    col = inp_f16.astype(np.float64)
    acc = col[..., :3].copy()
    n = float(p.samples)
    for i in range(p.samples + 1):
        uv = start * (1.0 - i / n) + end * (i / n)
        acc += np_bilinear(inp_f16, uv[..., 0], uv[..., 1])[..., :3]
    out = np.concatenate([acc / (n + 2.0), col[..., 3:4]], -1)
    return np.where(moved[..., None], out, col)


@pytest.mark.parametrize("frame,res", [(7, None), (0, None), (33, (130, 70))])
def test_motion_blur_oracle_matches_numpy_restatement(frame, res):
    H, W = 48, 80
    rng = np.random.default_rng(5)
    depth = rng.random((H, W)).astype(np.float32)
    vel = ch.rotation_velocity_field(W, H, depth)
    col = (rng.random((H, W, 4)) * 2.0).astype(np.float16)
    p = ch.motion_blur_params(W, H, frame=frame, resolution=res)
    inp = ch.make_inputs(32, 16, 1)
    got = orc.motion_blur(p, vel, col, inp.blue).astype(np.float64)
    want = np_motion_blur(p, vel, col, inp.blue)
    assert _agree(want, got, 2e-3, 1e-4, 2e-3) < 2e-3 and (got[:8, :8] == col[:8, :8].astype(np.float64)).all()


def np_hbao(p: abi.HbaoParams, depth, blue, prev, paths: dict | None = None):
    """hbao.frag:21-96 + hbao_utils.glsl (normal from depth, the spp-sample form: blueNoise() returns the same texel for every sample).
    paths: filled with the foreground pixels' `deltaDepth < th` ("near") and sample weight theta ("theta")"""
    H, W = depth.shape
    M = lambda arr: np.asarray(list(arr), np.float64).reshape(4, 4).T  # noqa: E731
    PV, Pinv, Mw = M(p.projection_view), M(p.projection_inverse), M(p.camera_matrix_world)
    ys, xs = np.mgrid[0:H, 0:W]
    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    d = depth.astype(np.float64)

    def world(dd, uu, vv):  # getWorldPos  hbao_utils.glsl:19-29
        clip = np.stack([uu * 2.0 - 1.0, vv * 2.0 - 1.0, dd * 2.0 - 1.0, np.ones_like(dd)], -1)
        w = (clip @ Pinv.T) @ Mw.T
        return w[..., :3] / w[..., 3:4]

    tap = lambda dx, dy: d[np.clip(ys + dy, 0, H - 1), np.clip(xs + dx, 0, W - 1)]  # noqa: E731  texelFetch, clamped
    c0, l2, l1, r1, r2, b2, b1, t1, t2 = tap(0, 0), tap(-2, 0), tap(-1, 0), tap(1, 0), tap(2, 0), tap(0, -2), tap(0, -1), tap(0, 1), tap(0, 2)
    dl, dr, db, dt = np.abs((2 * l1 - l2) - c0), np.abs((2 * r1 - r2) - c0), np.abs((2 * b1 - b2) - c0), np.abs((2 * t1 - t2) - c0)
    ce = world(c0, u, v)
    dpdx = np.where((dl < dr)[..., None], ce - world(l1, u - 1.0 / W, v), -ce + world(r1, u + 1.0 / W, v))
    dpdy = np.where((db < dt)[..., None], ce - world(b1, u, v - 1.0 / H), -ce + world(t1, u, v + 1.0 / H))
    n = np_normalize(np.cross(dpdx, dpdy))
    cam = Mw[:3, 3]
    bn = np_blue_noise(blue, p.blue_noise_index, W, H)
    r_, th_ = np.sqrt(bn[..., 0]), 2.0 * np.pi * bn[..., 1]
    b_ = np_normalize(np.cross(n, np.broadcast_to(np.array([0.0, 1.0, 1.0]), n.shape)))
    t_ = np.cross(b_, n)
    sdir = np_normalize((r_ * np.sin(th_))[..., None] * b_ + np.sqrt(1.0 - bn[..., 0])[..., None] * n + (r_ * np.cos(th_))[..., None] * t_)
    spos = ce + (p.ao_distance * np.power(bn[..., 2], p.distance_power + 1.0))[..., None] * sdir
    suv = np.concatenate([spos, np.ones((H, W, 1))], -1) @ PV.T
    su, sv = suv[..., 0] / suv[..., 3] * 0.5 + 0.5, suv[..., 1] / suv[..., 3] * 0.5 + 0.5
    sdepth = np_nearest(depth, su, sv).astype(np.float64)
    dist = np.linalg.norm(spos - cam, axis=-1)
    delta = (d - sdepth) * 0.001 * dist * dist
    th = p.thickness * 0.01
    theta = _dot(n, sdir)
    occ = np.sqrt(10.0 * np.maximum(0.0, sdepth + delta * p.bias * 1000.0 - d) * theta * np.maximum(0.0, 1.0 - delta / th) / dist)
    occ = np.where(delta < th, occ, 0.0)
    if paths is not None:
        fg = depth != 1.0
        paths.update(near=(delta < th)[fg], theta=theta[fg], blue_x=np.round(bn[..., 0] * 255.0)[fg])
    total = p.spp * theta
    ao = p.spp * occ
    ao = np.where(total > 0.0, ao / np.where(total == 0.0, 1.0, total), ao)
    out = np.concatenate([n, np.clip(1.0 - ao, 0.0, 1.0)[..., None]], -1)
    return np.where((depth == 1.0)[..., None], prev.astype(np.float64), out)


def test_hbao_oracle_matches_numpy_restatement():
    inp = ch.make_inputs(96, 64, 2)
    fr = inp.frames[1]
    p = ch.hbao_params(fr["cam"], 4242)
    prev = np.zeros((64, 96, 4), np.float16)
    got = orc.hbao(p, fr["depth"], inp.blue, prev).astype(np.float64)
    want = np_hbao(p, fr["depth"], inp.blue, prev)
    # fp16 target; the normal reconstruction picks the smoother side by comparing depth differences (dl < dr), which can flip at
    # silhouettes between fp32 and fp64, and so can the nearest depth tap of the sample
    assert _agree(want, got, 1e-3, 1e-3, 5e-3) < 5e-3   # (measured: 1 pixel of 6144)
    geo = fr["depth"] < 1.0
    assert (got[geo][:, 3] < 0.99).any() and (got[~geo] == 0.0).all()


def test_ssgi_compose_oracle_matches_numpy_restatement():
    rng = np.random.default_rng(6)
    H, W = 20, 36
    depth = rng.random((H, W)).astype(np.float32)
    depth[rng.random((H, W)) < 0.3] = 1.0
    gi = (rng.random((H, W, 4)) * 4).astype(np.float32)
    scene = (rng.random((H, W, 4)) * 4).astype(np.float16)
    got = orc.ssgi_compose(depth, gi, scene).astype(np.float64)   # ssgi_compose.frag:20-44 without fog: background -> scene colour, else the GI
    want = np.where((depth == 1.0)[..., None], scene[..., :3].astype(np.float64), gi[..., :3].astype(np.float64))
    _agree(want, got[..., :3], 1e-3, 1e-6, 0.0)
    assert (got[..., 3] == 1.0).all()


def test_env_cdf_tables_match_a_loop_for_loop_restatement():
    """synth.build_env_cdf (vectorised; it feeds rfx_env_set) against a statement-by-statement Python walk of gatherData
    (src/ssgi/utils/EquirectHdrInfoUniform.js:149-245): Float32Array stores, double accumulators, the lower-bound binary search."""
    from realism_effects_b200 import synth

    rng = np.random.default_rng(11)
    h, w = 8, 16
    data = (rng.random((h, w, 4)) ** 4 * 20.0).astype(np.float32)
    data[3] = 0.0                      # an all-black row: its conditional CDF stays unnormalised (all zeros)
    f32 = np.float32
    pdf_c, cdf_c, cdf_m = np.zeros(h * w, f32), np.zeros(h * w, f32), np.zeros(h, f32)
    total, cum_m = 0.0, 0.0
    for y in range(h):
        cum = 0.0
        for x in range(w):
            wgt = 0.2126 * float(data[y, x, 0]) + 0.7152 * float(data[y, x, 1]) + 0.0722 * float(data[y, x, 2])
            cum += wgt
            total += wgt
            pdf_c[y * w + x], cdf_c[y * w + x] = f32(wgt), f32(cum)
        if cum != 0:
            for i in range(y * w, y * w + w):
                cdf_c[i] = f32(float(cdf_c[i]) / cum)
        cum_m += cum
        cdf_m[y] = f32(cum_m)
    if cum_m != 0:
        for i in range(h):
            cdf_m[i] = f32(float(cdf_m[i]) / cum_m)

    def closest(arr, target, offset, count):
        lower, upper = offset, offset + count - 1
        while lower < upper:
            mid = (lower + upper) >> 1
            if float(arr[mid]) < target:
                lower = mid + 1
            else:
                upper = mid
        return lower - offset

    marg = np.array([(closest(cdf_m, (i + 1) / h, 0, h) + 0.5) / h for i in range(h)], f32)
    cond = np.array([[(closest(cdf_c, (x + 1) / w, y * w, w) + 0.5) / w for x in range(w)] for y in range(h)], f32)
    m2, c2, t2 = synth.build_env_cdf(data)
    assert np.array_equal(m2, marg) and np.array_equal(c2, cond) and abs(t2 - total) <= 1e-9 * total


def test_traa_form_of_temporal_reproject_matches_numpy_restatement():
    """K2 as TRAAEffect drives it (src/traa/TRAAEffect.js:21-31): one RGBA16F plane, inputType DIFFUSE, no discard, maxBlend 0.9,
    neighborhoodClampIntensity 1, confidencePower 4; the history here is last frame's colour buffer with alpha = a history length."""
    inp = ch.make_inputs(96, 64, 3)
    f0, f1 = inp.frames[1], inp.frames[2]
    p = ch.traa_temporal_params(abi.make_camera(f1["cam"]), f1["cam"]["position"], f0["cam"], 1.0)
    hist = f0["direct"].copy()
    hist[..., 3] = np.float16(3.0)
    z = np.zeros((64, 96, 4), np.float16)
    got, _ = orc.temporal_reproject(p, f1["direct"], f1["velocity"], hist, None, z, None, out_half=True)
    (want,) = np_temporal(p, f1["direct"], f1["velocity"], [hist], [z])
    assert _agree(want, got.astype(np.float64), 2e-3, 1e-4, 5e-3) < 5e-3
    assert (got[..., 3].astype(np.float64) > 0.5).mean() > 0.3   # history was blended in on a good part of the frame
