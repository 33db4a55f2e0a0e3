"""Drives the same synthetic frames through (a) the CUDA engine via the C ABI and (b) the CPU
oracle, pass by pass, following the reference's frame logic (SSGIEffect.update ->
SSGIPass.render -> Denoiser.render).  TEST INFRASTRUCTURE (imports tests/orc.py).

The oracle chain below is written in Python straight from the reference JS
(src/ssgi/pass/SSGIPass.js:68-95, src/temporal-reproject/TemporalReprojectPass.js:162-214,
src/denoise/pass/PoissonDenoisePass.js:135-149, src/denoise/Denoiser.js:97-107,
src/utils/BlueNoiseUtils.js:17-33) independently of the native chain in csrc/rfx_api.cu, so a
chain-level comparison also checks the native frame-state logic.
"""
from __future__ import annotations

import math
import os
import sys
from dataclasses import dataclass

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from realism_effects_b200 import abi, synth  # noqa: E402

RTOL, ATOL = 1e-3, 1e-5  # north_star: within 1e-3 relative per channel (ATOL guards exact zeros)


@dataclass
class Opts:
    """SSGI options (defaults = src/ssgi/SSGIOptions.js:26-48)."""

    distance: float = 10.0
    thickness: float = 10.0
    denoise_iterations: int = 1
    radius: float = 3.0
    phi: float = 0.5
    luma_phi: float = 5.0
    depth_phi: float = 2.0
    normal_phi: float = 50.0
    roughness_phi: float = 50.0
    specular_phi: float = 50.0
    env_blur: float = 0.5
    importance_sampling: bool = True
    steps: int = 20
    refine_steps: int = 5
    missed_rays: bool = False
    use_direct_light: bool = True
    use_envmap: bool = True
    mode: int = abi.MODE_SSGI
    blue_noise_start: int = 1234567
    resolution_scale: float = 1.0  # SSGIPass.js:53: only the SSGI target is scaled
    denoise_mode: int = 0  # Denoiser.js:7: 0 "full", 1 "full_temporal" (no Poisson pass), 2 "temporal" (no Poisson pass, no compose)

    @property
    def flags(self) -> int:
        f = 0
        if self.importance_sampling and self.use_envmap:
            f |= abi.SSGI_IMPORTANCE_SAMPLING
        if self.missed_rays:
            f |= abi.SSGI_MISSED_RAYS
        if self.use_direct_light:
            f |= abi.SSGI_USE_DIRECT_LIGHT
        if self.use_envmap:
            f |= abi.SSGI_USE_ENVMAP
        return f


@dataclass
class Inputs:
    width: int
    height: int
    frames: list  # of dicts of numpy planes + camera uniforms
    env_map: np.ndarray
    env_marginal: np.ndarray
    env_conditional: np.ndarray
    env_total: float
    blue: np.ndarray


def make_inputs(width: int, height: int, n_frames: int, *, static=False, env_size=(128, 64), device="cpu", reference_env=False, fov: float = 40.0,
                cam_step=(0.02, 0.0, 0.0), orthographic: bool = False, view_offset=None, blue_size: int = 128) -> Inputs:
    """reference_env: use the reference demo's environment map (synth.load_reference_env, SURVEY.md §8d) instead of the small analytic sky.
    orthographic: the same planes seen through a three.js OrthographicCamera (the shaders' #else branches of PERSPECTIVE_CAMERA): the projection
    matrices are replaced (Matrix4.makeOrthographic), the depth plane is re-encoded so that the view-space z of every texel is kept, and the
    camera dict carries perspective=False (abi.make_camera reads it).
    view_offset: a perspective camera's setViewOffset, called per frame (synth.render_frame), e.g. r2_jitter() or off_axis().
    blue_size: the blue-noise texture is the top-left blue_size x blue_size crop of the 128 x 128 asset (not a power of two: the
    kernels' `%` addressing)."""
    frames = []
    for t in range(n_frames):
        fr = synth.render_frame(width, height, t, device=device, static=static, fov=fov, cam_step=cam_step, view_offset=view_offset)
        u = fr.cam.uniforms()
        moved = (t > 0) and not static
        if orthographic:
            fr.depth = _to_orthographic(u, fr.depth, width / height)
        frames.append(dict(depth=fr.depth.cpu().numpy(), gbuffer=fr.gbuffer.cpu().numpy(), velocity=fr.velocity.cpu().numpy(),
                           direct=fr.direct_light.cpu().numpy(), cam=u, moved=moved))
    if reference_env:
        img, env = synth.load_reference_env()
        marg, cond, total = synth.build_env_cdf(img.astype(np.float32), flip_y=True)
    else:
        env = synth.synthetic_env(*env_size)
        marg, cond, total = synth.build_env_cdf(env.astype(np.float32), flip_y=False)
    return Inputs(width, height, frames, env, marg, cond, total, np.ascontiguousarray(synth.load_blue_noise()[:blue_size, :blue_size]))


def r2_jitter(width: int, height: int):
    """TRAA's sub-pixel jitter (effects.jitter: the R2 sequence, frame k's offset) as a make_inputs view_offset: projection[8] and [9]
    become small and non-zero"""
    from realism_effects_b200 import effects

    return lambda cam, k: effects.jitter(width, height, cam, k)


def off_axis(width: int, height: int):
    """the top-right width x height sub-rectangle of a 1.5x larger frame (setViewOffset, as a tiled or multi-monitor render takes it):
    projection[8] = 0.5 and projection[9] = 0.5, a strongly off-axis frustum"""
    return lambda cam, k: cam.setViewOffset(1.5 * width, 1.5 * height, 0.5 * width, 0.0, width, height)


def _to_orthographic(u: dict, depth, aspect: float, half_height: float = 11.0):
    """in place on the uniform dict `u`; returns the re-encoded depth plane (same torch dtype/device)"""
    n, f = float(u["near"]), float(u["far"])
    d = depth.double()
    view_z = (n * f) / ((f - n) * d - f)  # perspectiveDepthToViewZ
    od = (view_z + n) / (n - f)  # viewZToOrthographicDepth
    od = od.clamp(0.0, 1.0).where(d < 1.0, d)  # the background stays exactly 1.0
    top, right = half_height, half_height * aspect
    P = np.zeros((4, 4), np.float64)
    P[0, 0], P[1, 1], P[2, 2], P[2, 3], P[3, 3] = 1.0 / right, 1.0 / top, -2.0 / (f - n), -(f + n) / (f - n), 1.0
    u["projection"] = np.ascontiguousarray(P.T.reshape(16)).astype(np.float32)
    u["projection_inverse"] = np.ascontiguousarray(np.linalg.inv(P).T.reshape(16)).astype(np.float32)
    u["perspective"] = False
    return od.to(depth.dtype)


def next_blue(start: int, counter: int) -> int:
    """BlueNoiseUtils.js:25-28"""
    return (start + counter + 1) % 0x7FFFFFFF


def max_mip_level(w: int, h: int) -> float:
    return float(math.floor(math.log2(max(w, h))) + 1)  # Utils.js:30-34


def ssgi_params(o: Opts, cam: abi.CameraS, index: int, env_wh) -> abi.SsgiParams:
    p = abi.SsgiParams()
    p.cam = cam
    p.ray_distance, p.thickness, p.env_blur = o.distance, o.thickness, o.env_blur
    p.max_env_map_mip_level = max_mip_level(*env_wh) if o.use_envmap else 0.0
    p.steps, p.refine_steps, p.mode, p.flags, p.blue_noise_index = o.steps, o.refine_steps, o.mode, o.flags, index
    return p


def temporal_params(o: Opts, cam: abi.CameraS, cam_pos, prev: dict, keep_data: float, moved: bool) -> abi.TemporalParams:
    p = abi.TemporalParams()
    p.cam = cam
    abi.set_f16(p.prev_view_matrix, prev["view_matrix"])
    abi.set_f16(p.prev_camera_matrix_world, prev["camera_matrix_world"])
    abi.set_f16(p.prev_projection, prev["projection"])
    abi.set_f16(p.prev_projection_inverse, prev["projection_inverse"])
    p.camera_pos[:] = [float(x) for x in cam_pos]
    p.prev_camera_pos[:] = [float(x) for x in prev["position"]]
    p.max_blend, p.neighborhood_clamp_intensity, p.keep_data, p.confidence_power = 1.0, 0.5, keep_data, 0.75
    p.full_accumulate = 0 if moved else 1
    p.log_transform, p.history_linear = 1, 1
    if o.mode == abi.MODE_SSGI:
        p.texture_count, p.input_type = 2, abi.INPUT_DIFFUSE_SPECULAR
        p.reproject_specular[:] = [0, 1]
    else:
        p.texture_count, p.input_type = 1, abi.INPUT_SPECULAR
        p.reproject_specular[:] = [1, 1]
    return p


def poisson_params(o: Opts, index: int, first: bool) -> abi.PoissonParams:
    p = abi.PoissonParams()
    p.radius, p.phi, p.luma_phi, p.depth_phi, p.normal_phi = o.radius, o.phi, o.luma_phi, o.depth_phi, o.normal_phi
    p.roughness_phi, p.specular_phi = o.roughness_phi, o.specular_phi
    p.texture_count = 2 if o.mode == abi.MODE_SSGI else 1
    p.is_texture_specular[:] = [0, 1] if o.mode == abi.MODE_SSGI else [1, 1]
    p.gbuffer_texture, p.input_linear, p.blue_noise_index = 1, 0 if first else 1, index
    return p


def compose_params(cam: abi.CameraS, mode: int = abi.MODE_SSGI) -> abi.ComposeParams:
    p = abi.ComposeParams()
    p.cam = cam
    p.input_type = abi.INPUT_DIFFUSE_SPECULAR if mode == abi.MODE_SSGI else abi.INPUT_SPECULAR  # SSGIEffect.js:70-77
    return p


def chain_options(inp: Inputs, o: Opts) -> abi.ChainOptions:
    c = abi.ChainOptions()
    c.width, c.height = inp.width, inp.height
    c.denoise_iterations, c.steps, c.refine_steps = o.denoise_iterations, o.steps, o.refine_steps
    c.distance, c.thickness, c.env_blur = o.distance, o.thickness, o.env_blur
    c.radius, c.phi, c.luma_phi, c.depth_phi, c.normal_phi = o.radius, o.phi, o.luma_phi, o.depth_phi, o.normal_phi
    c.roughness_phi, c.specular_phi = o.roughness_phi, o.specular_phi
    c.ssgi_flags, c.mode, c.blue_noise_start = o.flags, o.mode, o.blue_noise_start
    c.denoise_mode = o.denoise_mode
    c.resolution_scale = o.resolution_scale
    return c


# ----------------------------------------------------------------------------------------------
def run_oracle_chain(inp: Inputs, o: Opts, capture=("ssgi", "tr0", "tr1", "dn0", "dn1", "composed"), lean: bool = False, impl=None):
    """Returns a list (one dict per frame) of the planes named in `capture` (+ the per-pass inputs
    needed for isolated kernel tests under keys starting with '_'; lean=True drops those copies: at 4K they are
    ~2.5 GB per frame).  `impl`: the module that executes the passes — tests/orc.py (the C++ restatement, default) or
    tests/refglsl.py (the reference's own shaders compiled for the CPU); both have the same pass signatures."""
    import orc as _orc

    orc = impl if impl is not None else _orc
    Env = _orc.Env  # the env tables / mip chain container is shared (host-built inputs of K1)

    H, W = inp.height, inp.width
    env = Env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total) if o.use_envmap else None
    z32 = lambda: np.zeros((H, W, 4), np.float32)  # noqa: E731
    z16 = lambda: np.zeros((H, W, 4), np.float16)  # noqa: E731
    tr = [z32(), z32()]
    dnA, dnB = [z16(), z16()], [z16(), z16()]
    composed = z32()
    fb = z32()  # denoiseMode != "full": the FramebufferTexture copy of the temporal target's attachment 0 (TemporalReprojectPass.js:134-152,197-200)
    keep_data, prev = 0.0, None
    bn_trace = bn_poisson = 0
    out = []
    for fr in inp.frames:
        cam = abi.make_camera(fr["cam"])
        rec = {}
        # K1
        bn_trace = next_blue(o.blue_noise_start, bn_trace)
        sp = ssgi_params(o, cam, bn_trace, (inp.env_map.shape[1], inp.env_map.shape[0]))
        rec["_k1_accumulated"] = composed.copy()
        rec["_k1_params"] = sp
        osz = None if o.resolution_scale == 1.0 else (int(W * o.resolution_scale), int(H * o.resolution_scale))
        ssgi = orc.ssgi_trace(sp, fr["depth"], fr["gbuffer"], None, fr["direct"], composed, env, inp.blue, out_size=osz)
        # K2
        if prev is None:
            prev = fr["cam"]
        tp = temporal_params(o, cam, fr["cam"]["position"], prev, keep_data, fr["moved"])
        rec["_k2_params"], rec["_k2_hist"], rec["_k2_prev_out"] = tp, [dnB[0].copy(), dnB[1].copy()], [tr[0].copy(), tr[1].copy()]
        if o.denoise_mode == 0:
            tr0, tr1 = orc.temporal_reproject(tp, ssgi, fr["velocity"], dnB[0], dnB[1], tr[0], tr[1])
        else:  # no denoise pass => overrideAccumulatedTextures is empty: BOTH accumulated textures are the one FramebufferTexture
            tr0, tr1 = orc.temporal_reproject(tp, ssgi, fr["velocity"], fb, fb, tr[0], tr[1])
            fb = tr0.copy()  # copyFramebufferToTexture after the draw (:197-200)
        tr = [tr0, tr1]
        keep_data, prev = 1.0, fr["cam"]
        if o.denoise_mode != 0:
            cp = compose_params(cam, o.mode)
            if o.denoise_mode == 1:  # "full_temporal": DenoiserComposePass on the temporal textures (Denoiser.js:55-64)
                if o.mode == abi.MODE_SSGI:
                    composed = orc.gi_compose(cp, fr["depth"], fr["gbuffer"], tr[0], tr[1], composed)
                else:
                    composed = orc.gi_compose(cp, fr["depth"], fr["gbuffer"], None, tr[0], composed, scene=fr["direct"])
            else:  # "temporal": denoiser.texture is the temporal pass's first texture (Denoiser.js:73-74); it is what K1 samples next frame
                composed = tr[0].copy()
            full = dict(ssgi=ssgi, tr0=tr[0], tr1=tr[1], dn0=dnB[0], dn1=dnB[1], composed=composed)
            out.append({k: full[k].copy() for k in capture})
            continue
        # K3
        rec["_k3"] = []
        for i in range(2 * o.denoise_iterations):
            horizontal = i % 2 == 0
            src = tr if i == 0 else (dnB if horizontal else dnA)
            dst = dnA if horizontal else dnB
            bn_poisson = next_blue(o.blue_noise_start, bn_poisson)
            pp = poisson_params(o, bn_poisson, i == 0)
            rec["_k3"].append(dict(params=pp, in0=src[0].copy(), in1=src[1].copy(), prev0=dst[0].copy(), prev1=dst[1].copy()))
            o0, o1 = orc.poisson_denoise(pp, fr["depth"], fr["gbuffer"], src[0], src[1], inp.blue, dst[0], dst[1])
            rec["_k3"][-1].update(out0=o0, out1=o1)
            if horizontal:
                dnA = [o0, o1]
            else:
                dnB = [o0, o1]
        # K4
        cp = compose_params(cam, o.mode)
        rec["_k4_params"], rec["_k4_prev"] = cp, composed.copy()
        if o.mode == abi.MODE_SSGI:
            composed = orc.gi_compose(cp, fr["depth"], fr["gbuffer"], dnB[0], dnB[1], composed)
        else:  # SSR: specular GI = the single Poisson target, diffuse component = the scene colour (composer input buffer)
            composed = orc.gi_compose(cp, fr["depth"], fr["gbuffer"], None, dnB[0], composed, scene=fr["direct"])
        full = dict(ssgi=ssgi, tr0=tr[0], tr1=tr[1], dn0=dnB[0], dn1=dnB[1], composed=composed)
        if lean:
            rec = {}
        rec.update({k: full[k].copy() for k in capture})
        out.append(rec)
    return out


def run_cuda_chain(inp: Inputs, o: Opts, capture=("ssgi", "tr0", "tr1", "dn0", "dn1", "composed"), fast_math: bool = True):
    from realism_effects_b200 import engine

    ctx = engine.Context(0, inp.blue)
    ctx.set_fast_math(fast_math)
    try:
        if o.use_envmap:
            ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        chain = engine.SsgiChain(ctx, chain_options(inp, o))
        which = dict(composed=0, ssgi=1, tr0=2, tr1=3, dn0=4, dn1=5)
        out = []
        for fr in inp.frames:
            d, g, v, dl = ctx.upload(fr["depth"]), ctx.upload(fr["gbuffer"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            chain.render(abi.make_camera(fr["cam"]), d, g, v, dl, fr["cam"]["position"], fr["moved"])
            out.append({k: chain.download(which[k]) for k in capture})
            for p in (d, g, v, dl):
                p.free()
        launches = ctx.launch_count
        chain.close()
        return out, launches
    finally:
        ctx.close()


# ----------------------------------------------------------------------------------------------
def unpack_halves(a: np.ndarray) -> np.ndarray:
    """RGBA32F plane of packed half pairs -> (H,W,8) float32"""
    return a.view(np.uint32).view(np.float16).astype(np.float32).reshape(a.shape[0], a.shape[1], 8)


def compare(a: np.ndarray, b: np.ndarray, packed: bool = False, rtol: float | None = None) -> dict:
    """Per-channel |a-b| <= RTOL*max(|a|,|b|) + ATOL; returns max relative error over the
    conforming elements, the fraction of PIXELS with any non-conforming channel, and bit-equality."""
    if packed:
        a, b = unpack_halves(a), unpack_halves(b)
    a = a.astype(np.float64)
    b = b.astype(np.float64)
    fin = np.isfinite(a) & np.isfinite(b)
    same_nonfinite = (~fin) & ((a == b) | (np.isnan(a) & np.isnan(b)))
    diff = np.where(fin, np.abs(a - b), 0.0)
    scale = np.where(fin, np.maximum(np.abs(a), np.abs(b)), 0.0)
    bad = (diff > (RTOL if rtol is None else rtol) * scale + ATOL) | ((~fin) & ~same_nonfinite)
    rel = np.where(scale > 0, diff / np.maximum(scale, 1e-30), 0.0)
    ok_rel = np.where(bad, 0.0, rel)
    bad_px = bad.reshape(bad.shape[0], bad.shape[1], -1).any(-1)
    return dict(frac_bad=float(bad_px.mean()), n_bad=int(bad_px.sum()), max_rel_ok=float(ok_rel.max()), max_abs=float(diff.max()),
                bit_equal=float(((a == b) | (np.isnan(a) & np.isnan(b))).mean()))


def differing_pixels(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """(y, x) of the pixels whose bytes differ between two planes of one shape and dtype, in row-major order.  In an fp16 plane a channel
    that is NaN in both counts as equal whatever its sign and payload: neither IEEE arithmetic nor GLSL defines which NaN an invalid
    operation returns, and the host's libm (log of a negative number: -NaN on x86-64) and the device's (+NaN) differ there; the Poisson
    targets of the AO chain hold such NaNs in the channels ao_compose does not read.  fp32 planes are compared bit for bit: K1's packs
    two halves into one fp32 word, which must not count as a float NaN."""
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, a.dtype, b.shape, b.dtype)
    u = {1: np.uint8, 2: np.uint16, 4: np.uint32}[a.dtype.itemsize]
    d = a.view(u) != b.view(u)
    if a.dtype == np.float16:
        d &= ~(np.isnan(a) & np.isnan(b))
    return np.argwhere(d.reshape(a.shape[0], a.shape[1], -1).any(-1))


def byte_report(name: str, want: np.ndarray, got: np.ndarray) -> str:
    """'' when the planes are byte-equal, else how many pixels differ and the first one, with both values"""
    d = differing_pixels(want, got)
    if not len(d):
        return ""
    y, x = (int(v) for v in d[0])
    return f"{name}: {len(d)} pixels differ from the oracle, first at (y, x) = ({y}, {x}): oracle {want[y, x].tolist()} kernel {got[y, x].tolist()}"


def run_chain_parity(width=192, height=108, frames=2, fast_math=True, inputs_kw=None, **opt_kw) -> dict:
    o = Opts(**opt_kw)
    inp = make_inputs(width, height, frames, **(inputs_kw or {}))
    ref = run_oracle_chain(inp, o)
    got, launches = run_cuda_chain(inp, o, fast_math=fast_math)
    # The exact variant runs kernels that are each bit-equal to the oracle, so every plane of every frame must equal the oracle's byte
    # for byte.  The fast variant's SFU transcendentals differ from the oracle in the last bits; every pass of every frame re-quantises
    # to fp16 (K1 pack, Poisson targets), so such a difference in one pass can become a 1-fp16-ulp (<= 9.8e-4 relative) difference at
    # the next quantisation point.  Its bars (fraction of pixels with a channel outside the band, worst plane of any frame): 6e-3 outside
    # 1e-3 / 1.5e-3 outside 4e-3.  These small frames have ~2e4 pixels, so ONE march ray that resolves differently (its footprint after
    # the denoiser is ~50 pixels) is 2.5e-3 of a plane: the statistically meaningful bars (1e-3 / 2e-4 at 1080p and 4K) are in
    # tests/test_gpu_parity_at_size.py.
    loose_frac, max_frac = 6e-3, 1.5e-3
    worst, worst4, lines, differ = 0.0, 0.0, [], []
    ssr = o.mode == abi.MODE_SSR
    for t, (r, g) in enumerate(zip(ref, got)):
        for k in ("ssgi", "tr0", "tr1", "dn0", "dn1", "composed"):
            rep = byte_report(f"f{t}.{k}", r[k], g[k])
            if rep:
                differ.append(rep)
            if ssr and k == "ssgi":  # SSR: rgb fp32 + (rayLength, roughness) packed in alpha (ssgi.frag:302-308): compare the colour channels
                c, c4 = compare(r[k][..., :3], g[k][..., :3]), compare(r[k][..., :3], g[k][..., :3], rtol=4e-3)
                worst, worst4 = max(worst, c["frac_bad"]), max(worst4, c4["frac_bad"])
                lines.append(f"f{t}.{k}: bad={c['frac_bad']:.2e} bad@4e-3={c4['frac_bad']:.1e} biteq={c['bit_equal']:.4f}")
                continue
            c = compare(r[k], g[k], packed=(k == "ssgi"))
            c4 = compare(r[k], g[k], packed=(k == "ssgi"), rtol=4e-3)
            worst, worst4 = max(worst, c["frac_bad"]), max(worst4, c4["frac_bad"])
            lines.append(f"f{t}.{k}: bad={c['frac_bad']:.2e} bad@4e-3={c4['frac_bad']:.1e} biteq={c['bit_equal']:.4f}")
    if fast_math:
        ok = worst <= loose_frac and worst4 <= max_frac
        head = f"worst bad-pixel fraction {worst:.2e} at 1e-3 (limit {loose_frac:.0e}), {worst4:.2e} at 4e-3 (limit {max_frac:.0e}); "
    else:
        ok = not differ
        head = ("every plane of every frame byte-equal to the oracle; " if ok else "; ".join(differ) + "; ")
    return dict(ok=ok, worst=worst, worst4=worst4, launches=launches, differ=differ, summary=head + "; ".join(lines))


# ----------------------------------------------------------------------------------------------
# other passes: HBAO (C4), AO compose, motion blur (C1), TRAA
# ----------------------------------------------------------------------------------------------
def hbao_params(cam_u: dict, index: int, spp: int = 8) -> abi.HbaoParams:
    """defaults src/ao/AOEffect.js:8-21; projectionViewMatrix = projectionMatrix * matrixWorldInverse (AOPass.js:93-96),
    multiplied in float64 like three.js' Matrix4 (JS numbers) and uploaded as float32."""
    p = abi.HbaoParams()
    P = np.asarray(cam_u["projection"], np.float64).reshape(4, 4).T
    V = np.asarray(cam_u["view_matrix"], np.float64).reshape(4, 4).T
    abi.set_f16(p.projection_view, np.ascontiguousarray((P @ V).T.reshape(16)).astype(np.float32))
    abi.set_f16(p.projection_inverse, cam_u["projection_inverse"])
    abi.set_f16(p.camera_matrix_world, cam_u["camera_matrix_world"])
    p.ao_distance, p.distance_power, p.bias, p.thickness, p.spp, p.blue_noise_index = 2.0, 1.0, 40.0, 0.075, spp, index
    return p


def ao_compose_params(power: float = 2.0, color=(0.0, 0.0, 0.0)) -> abi.AoComposeParams:
    p = abi.AoComposeParams()
    p.power = power
    p.color[:] = list(color)
    return p


def motion_blur_params(width: int, height: int, frame: int = 7, samples: int = 16, delta_time: float = 1 / 60, resolution=None) -> abi.MotionBlurParams:
    """defaults src/motion-blur/MotionBlurEffect.js:14; `resolution` is the window size (may differ from the buffer size)."""
    p = abi.MotionBlurParams()
    p.intensity, p.jitter, p.delta_time = 1.0, 1.0, max(1 / 1000, delta_time)
    p.resolution[:] = list(resolution or (width, height))
    p.frame, p.samples = frame, samples
    return p


def rotation_velocity_field(width: int, height: int, depth: np.ndarray, vmax: float = 0.05) -> np.ndarray:
    """C1: rigid rotation about the image centre, |v| up to vmax in uv units; velocity-plane layout."""
    ys, xs = np.meshgrid((np.arange(height) + 0.5) / height - 0.5, (np.arange(width) + 0.5) / width - 0.5, indexing="ij")
    k = vmax / 0.5
    vel = np.zeros((height, width, 4), np.float32)
    vel[..., 0], vel[..., 1] = (-ys * k).astype(np.float32), (xs * k).astype(np.float32)
    vel[..., 3] = depth
    vel[:8, :8, :2] = 0.0  # a patch that did not move (early-out branch)
    return vel


def traa_temporal_params(cam: abi.CameraS, cam_pos, prev: dict, keep_data: float) -> abi.TemporalParams:
    """TRAAEffect forced options (src/traa/TRAAEffect.js:21-31) over the TemporalReprojectPass defaults (:17-32)."""
    p = abi.TemporalParams()
    p.cam = cam
    abi.set_f16(p.prev_view_matrix, prev["view_matrix"])
    abi.set_f16(p.prev_camera_matrix_world, prev["camera_matrix_world"])
    abi.set_f16(p.prev_projection, prev["projection"])
    abi.set_f16(p.prev_projection_inverse, prev["projection_inverse"])
    p.camera_pos[:] = [float(x) for x in cam_pos]
    p.prev_camera_pos[:] = [float(x) for x in prev["position"]]
    p.max_blend, p.neighborhood_clamp_intensity, p.keep_data, p.confidence_power = 0.9, 1.0, keep_data, 4.0
    p.full_accumulate, p.texture_count, p.input_type, p.log_transform, p.history_linear = 0, 1, abi.INPUT_DIFFUSE, 1, 1
    p.reproject_specular[:] = [0, 0]
    return p


# ----------------------------------------------------------------------------------------------
# pass sequences shared by the golden minting script (run on the reference shaders) and the tests (run on the oracle / the engine);
# `m` is the module that executes the passes (tests/refglsl.py, tests/orc.py)
# ----------------------------------------------------------------------------------------------
def fog_params(cam_u, exp2):
    p = abi.SsgiComposeParams()
    p.use_fog, p.fog_exp2, p.perspective = 1, int(exp2), 1
    p.fog_color[:] = [0.6, 0.7, 0.8]
    p.fog_near, p.fog_far, p.fog_density = 2.0, 30.0, 0.05
    p.camera_near, p.camera_far = float(cam_u["near"]), float(cam_u["far"])
    return p


def ao_denoise(m, f1, blue, ao):
    """AOEffect's denoiser: 2 Poisson passes over one plane with the velocity-layout normals (non-GBUFFER branch)"""
    H, W = f1["depth"].shape
    tgtA, tgtB = np.zeros((H, W, 4), np.float16), np.zeros((H, W, 4), np.float16)
    for i in range(2):
        p = poisson_params(Opts(), 1234568 + i, False)
        p.texture_count, p.gbuffer_texture, p.input_linear = 1, 0, 1
        p.is_texture_specular[:] = [0, 0]
        p.normal_phi, p.depth_phi, p.roughness_phi, p.specular_phi = 3.25, 2.0, 0.0, 0.0
        out, _ = m.poisson_denoise(p, f1["depth"], f1["velocity"], ao if i == 0 else tgtA, None, blue, tgtA if i == 0 else tgtB, None)
        if i == 0:
            tgtA = out
        else:
            tgtB = out
    return tgtA, tgtB


def traa_two_frames(m, f0, f1):
    z = np.zeros(f0["direct"].shape, np.float16)
    p0 = traa_temporal_params(abi.make_camera(f0["cam"]), f0["cam"]["position"], f0["cam"], 0.0)
    h0, _ = m.temporal_reproject(p0, f0["direct"], f0["velocity"], z, None, z, None, out_half=True)
    p1 = traa_temporal_params(abi.make_camera(f1["cam"]), f1["cam"]["position"], f0["cam"], 1.0)
    h1, _ = m.temporal_reproject(p1, f1["direct"], f1["velocity"], h0, None, h0, None, out_half=True)
    return h0, h1


FX_CASES = [  # (effects in EffectPass order, sparkle_perspective)
    ([abi.FX_SHARPNESS], False), ([abi.FX_LENS_DISTORTION], False), ([abi.FX_GRADUAL_BACKGROUND], False), ([abi.FX_SPARKLE], False), ([abi.FX_SPARKLE], True),
    ([abi.FX_SHARPNESS, abi.FX_GRADUAL_BACKGROUND, abi.FX_SPARKLE], False), ([abi.FX_LENS_DISTORTION, abi.FX_SHARPNESS], False),
]


def fx_params(cam_u, effects, sparkle_perspective=False):
    """non-default values where the default would saturate on the synthetic scene (GradualBackground's fade is 1 everywhere at maxDistance 5)"""
    return abi.make_effects_params(cam_u, effects, sharpness=1.5, background_color=(0.2, 0.3, 0.5), max_distance=20.5, sparkle_perspective=sparkle_perspective)


def taa_cases():
    out = []
    for n in (0.0, 1.0, 7.0):
        for srgb in (0, 1):
            p = abi.TaaParams()
            p.camera_not_moved_frames, p.srgb_output = n, srgb
            out.append(p)
    return out
