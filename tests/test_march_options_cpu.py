"""The SSGI march (K1) and the temporal reprojection (K2) across their option space, on the CPU: the case grid that
tests/test_gpu_march_options.py runs the CUDA kernels on, what kernel each case reaches, and the oracle against the reference's own
shaders (tests/refpins.py) at the grid's points, so that the kernels are held to the reference there.

K1 points: every value of (steps - 1) mod 4 (the fast march tests RFX_K1_BATCH = 4 steps per batch) and steps = 1 (no march at all);
refineSteps 0, 1 and 7; thickness and ray distance small enough that the hit test and the step length decide rays; env-blur 0 and 1; the
four flag sets; SSGI and SSR; a velocity plane, a missing direct-light plane, frame 0 (no accumulated plane), a smaller target
(resolutionScale 0.5 and 0.75); symmetric, TRAA-jittered, off-axis (projection[8] = projection[9] = 0.5) and orthographic cameras; an env
map whose mip chain has odd sizes (100 x 50 -> 50 x 25 -> 25 x 12 -> 12 x 6 -> 6 x 3 -> 3 x 1 -> 1 x 1) and a 96 x 96 blue-noise texture.
K2 points: the three forms (2 planes of packed diffuse + specular; 1 specular plane; 1 diffuse plane, TRAA's fp16 form), each switch of
TemporalArgs both ways, fp16 and fp32 history, a scaled input, and moving, static and off-axis cameras."""
from __future__ import annotations

from dataclasses import dataclass, replace

import numpy as np

import chain_harness as ch
import orc
import refpins
from realism_effects_b200 import abi

FLAGS = {  # flag set -> (importance_sampling, use_envmap, use_direct_light, missed_rays)
    "default": (True, True, True, False),
    "no-is": (False, True, True, False),
    "no-env-dl": (False, False, False, False),
    "missed": (True, True, True, True),
}
CAMERAS = ("sym", "jitter", "offaxis", "ortho")


@dataclass(frozen=True)
class K1Case:
    W: int = 200
    H: int = 120
    steps: int = 20
    refine: int = 5
    thickness: float = 10.0
    distance: float = 10.0
    env_blur: float = 0.5
    flags: str = "default"
    mode: int = abi.MODE_SSGI
    camera: str = "sym"
    env: tuple = (128, 64)
    blue: int = 128
    velocity: bool = False   # a velocity plane is bound (K1 subtracts its motion from the hit's uv)
    direct: bool = True      # the direct-light plane is bound (its flag may still be off)
    accumulated: bool = True  # false: frame 0, no accumulated plane
    scale: float = 1.0       # resolutionScale: the target is (int(W * scale), int(H * scale))

    def __str__(self):
        s = (f"{self.W}x{self.H}-{'ssr' if self.mode == abi.MODE_SSR else 'ssgi'}-s{self.steps}r{self.refine}-t{self.thickness:g}-d{self.distance:g}"
             f"-b{self.env_blur:g}-{self.flags}-{self.camera}")
        if self.env != (128, 64):
            s += f"-env{self.env[0]}x{self.env[1]}"
        if self.blue != 128:
            s += f"-blue{self.blue}"
        s += "".join(t for t, on in (("-vel", self.velocity), ("-nodl", not self.direct), ("-noacc", not self.accumulated)) if on)
        return s + (f"-scale{self.scale:g}" if self.scale != 1.0 else "")

    def opts(self, **kw) -> ch.Opts:
        is_, env, dl, missed = FLAGS[self.flags]
        return ch.Opts(steps=self.steps, refine_steps=self.refine, thickness=self.thickness, distance=self.distance, env_blur=self.env_blur,
                       importance_sampling=is_, use_envmap=env, use_direct_light=dl, missed_rays=missed, mode=self.mode,
                       resolution_scale=self.scale, **kw)


K1_CASES = [
    K1Case(),
    K1Case(steps=1, refine=0, thickness=0.5, env_blur=0.0, camera="offaxis"),
    K1Case(203, 117, steps=2, refine=1, thickness=0.05, distance=40.0, env_blur=1.0, flags="no-is", camera="offaxis", env=(100, 50)),
    K1Case(90, 160, steps=3, refine=7, distance=0.5, flags="missed", mode=abi.MODE_SSR, camera="offaxis"),
    K1Case(13, 9, steps=4, refine=0, thickness=0.5, flags="no-env-dl", camera="jitter", accumulated=False),
    K1Case(17, 33, steps=5, refine=1, distance=40.0, env_blur=1.0, mode=abi.MODE_SSR, camera="jitter", env=(100, 50), blue=96),
    K1Case(steps=33, refine=7, thickness=0.05, camera="ortho"),
    K1Case(203, 117, refine=0, thickness=0.5, distance=40.0, flags="missed", camera="offaxis", blue=96, velocity=True),
    K1Case(90, 160, steps=33, refine=1, env_blur=0.0, flags="no-is", mode=abi.MODE_SSR, camera="ortho"),
    K1Case(steps=5, refine=7, thickness=0.5, distance=0.5, scale=0.5),
    K1Case(203, 117, steps=4, refine=1, camera="offaxis", env=(100, 50), scale=0.75),
    K1Case(steps=2, thickness=0.05, mode=abi.MODE_SSR, camera="offaxis", direct=False, accumulated=False),
    K1Case(17, 33, steps=3, refine=0, flags="no-is", camera="ortho", velocity=True),
    K1Case(13, 9, refine=1, env_blur=1.0, mode=abi.MODE_SSR, camera="ortho", env=(100, 50)),
    K1Case(90, 160, steps=1, flags="missed", mode=abi.MODE_SSR, camera="jitter"),
    K1Case(203, 117, steps=5, refine=0, thickness=0.05, flags="no-env-dl", mode=abi.MODE_SSR, camera="jitter"),
    K1Case(steps=33, refine=0, distance=40.0, camera="jitter", env=(100, 50)),
]


def make_inputs(W: int, H: int, camera: str = "sym", env=(128, 64), blue: int = 128, frames: int = 2, static: bool = False) -> ch.Inputs:
    vo = {"jitter": ch.r2_jitter(W, H), "offaxis": ch.off_axis(W, H)}.get(camera)
    return ch.make_inputs(W, H, frames, env_size=env, blue_size=blue, orthographic=camera == "ortho", view_offset=vo, static=static)


def accumulated_plane(W: int, H: int, seed: int) -> np.ndarray:
    """last frame's `composed` as K1 samples it: colours in [0, 2), alpha 1"""
    a = np.random.default_rng(seed).uniform(0.0, 2.0, (H, W, 4)).astype(np.float32)
    a[..., 3] = 1.0
    return a


def k1_call(case: K1Case, inp: ch.Inputs, index: int):
    """the arguments of one K1 call on frame 1 of `inp`: (params, depth, gbuffer, velocity, direct, accumulated, env or None, out_size)"""
    fr = inp.frames[1]
    o = case.opts()
    p = ch.ssgi_params(o, abi.make_camera(fr["cam"]), index, (inp.env_map.shape[1], inp.env_map.shape[0]))
    env = orc.Env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total) if o.use_envmap else None
    out_size = None if case.scale == 1.0 else (int(inp.width * case.scale), int(inp.height * case.scale))
    return (p, fr["depth"], fr["gbuffer"], fr["velocity"] if case.velocity else None, fr["direct"] if case.direct else None,
            accumulated_plane(inp.width, inp.height, index) if case.accumulated else None, env, out_size)


def proj_sparse(projection) -> bool:
    """rfx_api.cu's test for the perspective sparsity pattern (column-major m[col * 4 + row]); m[8] and m[9] may be anything"""
    M = np.asarray(projection, np.float32)
    return bool(all(M[i] == 0.0 for i in (1, 2, 3, 4, 6, 7, 12, 13, 15)) and M[11] == -1.0)


def k1_path(case: K1Case, fast: bool, projection) -> tuple:
    """(kernel, mode, importance sampling, sparse projection, scaled target) of launch_ssgi / launch_ssgi_t: the fused fast kernel
    addresses texels by pixel index, so a smaller target takes the general kernel even with fast math on"""
    o = case.opts()
    scaled = case.scale != 1.0 and (int(case.W * case.scale) != case.W or int(case.H * case.scale) != case.H)
    kernel = "ssgi_fast_kernel" if fast and not scaled else "ssgi_kernel"
    return kernel, o.mode, bool(o.flags & abi.SSGI_IMPORTANCE_SAMPLING), proj_sparse(projection), scaled


@dataclass(frozen=True)
class K2Case:
    W: int = 200
    H: int = 120
    form: str = "ssgi"  # "ssgi": 2 planes, packed diffuse + specular input; "ssr": 1 specular plane; "traa": 1 diffuse plane, fp16 in and out
    camera: str = "moving"  # "moving", "static" (full accumulation: no camera motion) or "offaxis" (moving)
    log_transform: int = 1
    full_accumulate: int = 0
    keep_data: float = 1.0
    history_linear: int = 1
    hist32: bool = False  # the RGBA32F history of denoiseMode "full_temporal" / "temporal"
    scale: float = 1.0    # the input is K1's smaller target (resolutionScale)
    confidence_power: float = 0.75
    max_blend: float = 1.0
    clamp: float = 0.5
    rs: tuple = (0, 1)

    def __str__(self):
        return (f"{self.W}x{self.H}-{self.form}-{self.camera}-log{self.log_transform}-fa{self.full_accumulate}-keep{self.keep_data:g}"
                f"-lin{self.history_linear}-h{32 if self.hist32 else 16}-cp{self.confidence_power:g}-mb{self.max_blend:g}-cl{self.clamp:g}"
                f"-rs{''.join(map(str, self.rs))}" + (f"-scale{self.scale:g}" if self.scale != 1.0 else ""))

    @property
    def texture_count(self) -> int:
        return 2 if self.form == "ssgi" else 1

    @property
    def input_type(self) -> int:
        return {"ssgi": abi.INPUT_DIFFUSE_SPECULAR, "ssr": abi.INPUT_SPECULAR, "traa": abi.INPUT_DIFFUSE}[self.form]


K2_CASES = [
    K2Case(),
    K2Case(203, 117, camera="static", log_transform=0, full_accumulate=1, history_linear=0, confidence_power=0.125, max_blend=0.5, clamp=0.0, rs=(1, 0)),
    K2Case(90, 160, camera="offaxis", keep_data=0.0, hist32=True, confidence_power=4.0, max_blend=0.9, clamp=1.0, rs=(1, 0)),
    K2Case(full_accumulate=1, history_linear=0, scale=0.5, confidence_power=1.0, max_blend=0.9),
    K2Case(203, 117, form="ssr", log_transform=0, history_linear=0, hist32=True, confidence_power=4.0, max_blend=0.5, clamp=1.0, rs=(1,)),
    K2Case(90, 160, form="ssr", camera="offaxis", keep_data=0.0, full_accumulate=1, confidence_power=0.125, clamp=0.0, rs=(1,)),
    K2Case(form="ssr", camera="static", scale=0.75, rs=(1,)),
    K2Case(form="traa", confidence_power=4.0, max_blend=0.9, clamp=1.0, rs=(0,)),
    K2Case(203, 117, form="traa", camera="static", log_transform=0, history_linear=0, keep_data=0.0, rs=(0,)),
    K2Case(90, 160, form="traa", camera="offaxis", hist32=True, full_accumulate=1, confidence_power=1.0, max_blend=0.5, clamp=0.0, rs=(0,)),
    K2Case(203, 117, camera="offaxis", log_transform=0, hist32=True, keep_data=0.0, confidence_power=1.0, clamp=1.0),
]


def k2_inputs(case: K2Case) -> ch.Inputs:
    return make_inputs(case.W, case.H, "offaxis" if case.camera == "offaxis" else "sym", static=case.camera == "static")


def k2_call(case: K2Case, inp: ch.Inputs):
    """one K2 call on frame 1 of `inp`: (params, input, velocity, history0, history1, target0, target1, out_half).  The SSGI / SSR forms
    take frame 1 of the oracle's chain (its K1 plane, its denoised planes or its last temporal planes as history); TRAA takes the direct
    light of frames 1 and 0."""
    f0, f1 = inp.frames
    if case.form == "traa":
        p = ch.traa_temporal_params(abi.make_camera(f1["cam"]), f1["cam"]["position"], f0["cam"], case.keep_data)
        hist = f0["direct"].astype(np.float32) if case.hist32 else f0["direct"]
        args = [f1["direct"], f1["velocity"], hist, None, np.zeros_like(f1["direct"]), None, True]
    else:
        o = ch.Opts(mode=abi.MODE_SSGI if case.form == "ssgi" else abi.MODE_SSR, resolution_scale=case.scale, steps=8, refine_steps=3)
        rec = ch.run_oracle_chain(inp, o, capture=("ssgi",))[1]
        p = rec["_k2_params"]
        hist = rec["_k2_prev_out"] if case.hist32 else rec["_k2_hist"]
        two = case.texture_count == 2
        args = [rec["ssgi"], f1["velocity"], hist[0], hist[1] if two else None, rec["_k2_prev_out"][0], rec["_k2_prev_out"][1] if two else None, False]
    p.texture_count, p.input_type = case.texture_count, case.input_type
    p.log_transform, p.full_accumulate, p.keep_data, p.history_linear = case.log_transform, case.full_accumulate, case.keep_data, case.history_linear
    p.confidence_power, p.max_blend, p.neighborhood_clamp_intensity = case.confidence_power, case.max_blend, case.clamp
    p.reproject_specular[:] = list(case.rs) + [0] * (2 - len(case.rs))
    return [p] + args


def k2_switches(case: K2Case) -> dict:
    """the K2 kernel's switches (TemporalArgs) this case sets"""
    return dict(texture_count=case.texture_count, input_type=case.input_type, input_half=case.form == "traa", out_half=case.form == "traa",
                log_transform=case.log_transform, full_accumulate=case.full_accumulate, keep_data=case.keep_data, history_linear=case.history_linear,
                hist_f32=case.hist32, in_scaled=case.scale != 1.0, rs0=case.rs[0], rs1=case.rs[1] if len(case.rs) > 1 else None,
                moving=case.camera != "static")


# ---- coverage ------------------------------------------------------------------------------------------------------------------------
_inputs: dict = {}


def cached_inputs(key: tuple) -> ch.Inputs:
    if key not in _inputs:
        _inputs[key] = make_inputs(*key)
    return _inputs[key]


def k1_inputs(case: K1Case) -> ch.Inputs:
    return cached_inputs((case.W, case.H, case.camera, case.env, case.blue))


def test_k1_grid_reaches_every_kernel_path():
    """both kernels x MODE x IS x SPARSE, the scaled general path, every (steps - 1) mod 4 and steps = 1, refineSteps 0 and above,
    and each listed value of every option at least once"""
    paths = set()
    for c in K1_CASES:
        inp = k1_inputs(c)
        for fr in inp.frames:
            assert 0.0 < (fr["depth"] == 1.0).mean() < 1.0, str(c)  # background next to shaded pixels
        for fast in (True, False):
            paths.add(k1_path(c, fast, inp.frames[1]["cam"]["projection"]))
    reached = {(k, m, i, s) for k, m, i, s, scaled in paths if not scaled}
    want = {(k, m, i, s) for k in ("ssgi_fast_kernel", "ssgi_kernel") for m in (abi.MODE_SSGI, abi.MODE_SSR) for i in (False, True) for s in (False, True)}
    assert reached == want, want - reached
    assert {(k, scaled) for k, _, _, _, scaled in paths} == {("ssgi_fast_kernel", False), ("ssgi_kernel", False), ("ssgi_kernel", True)}
    assert {(c.steps - 1) % 4 for c in K1_CASES if c.steps > 1} == {0, 1, 2, 3} and any(c.steps == 1 for c in K1_CASES)
    assert {c.steps for c in K1_CASES} == {1, 2, 3, 4, 5, 20, 33}
    assert {c.refine for c in K1_CASES} == {0, 1, 5, 7}
    assert any(c.refine == 0 and c.flags == "default" and c.direct for c in K1_CASES)  # refine 0 with an env map and direct light
    assert {c.thickness for c in K1_CASES} == {0.05, 0.5, 10.0} and {c.distance for c in K1_CASES} == {0.5, 10.0, 40.0}
    assert {0.0, 1.0} <= {c.env_blur for c in K1_CASES}
    assert {c.flags for c in K1_CASES} == set(FLAGS) and {c.camera for c in K1_CASES} == set(CAMERAS)
    assert {(c.W, c.H) for c in K1_CASES} == {(200, 120), (203, 117), (90, 160), (13, 9), (17, 33)}
    assert {c.env for c in K1_CASES} == {(128, 64), (100, 50)} and {c.blue for c in K1_CASES} == {128, 96}
    assert {c.scale for c in K1_CASES} == {1.0, 0.5, 0.75}
    assert any(c.velocity for c in K1_CASES) and any(not c.direct for c in K1_CASES) and any(not c.accumulated for c in K1_CASES)
    assert any(c.env == (100, 50) and FLAGS[c.flags][0] for c in K1_CASES)  # odd mip levels under importance sampling
    for cam in ("jitter", "offaxis"):  # the terms the sparse path keeps are non-zero, and large for the off-axis camera
        P = make_inputs(200, 120, cam).frames[1]["cam"]["projection"]
        assert P[8] != 0.0 and P[9] != 0.0 and proj_sparse(P)
        assert (min(abs(P[8]), abs(P[9])) > 0.4) == (cam == "offaxis")


def test_k2_grid_takes_every_switch_both_ways():
    sw = [k2_switches(c) for c in K2_CASES]
    for k in sw[0]:
        vals = {s[k] for s in sw if s[k] is not None}
        assert len(vals) >= 2, (k, vals)
    assert {(s["texture_count"], s["input_type"]) for s in sw} == {(2, abi.INPUT_DIFFUSE_SPECULAR), (1, abi.INPUT_SPECULAR), (1, abi.INPUT_DIFFUSE)}
    assert {(c.rs) for c in K2_CASES if c.form == "ssgi"} == {(0, 1), (1, 0)}
    assert {c.confidence_power for c in K2_CASES} == {0.125, 0.75, 1.0, 4.0}
    assert {c.max_blend for c in K2_CASES} == {0.5, 0.9, 1.0} and {c.clamp for c in K2_CASES} == {0.0, 0.5, 1.0}
    assert {c.camera for c in K2_CASES} == {"moving", "static", "offaxis"}
    assert {c.form for c in K2_CASES if c.hist32} == {"ssgi", "ssr", "traa"}


# ---- the oracle against the reference's shaders --------------------------------------------------------------------------------------
PIN_SIZES = {(200, 120): (64, 40), (203, 117): (57, 33), (90, 160): (24, 40), (13, 9): (13, 9), (17, 33): (17, 33)}


def test_oracle_equals_reference_shaders_march_options():
    """every K1 and K2 case of the grid at a frame of 64 x 40 or smaller: the oracle's outputs, bit for bit"""
    R = refpins.ref("march_options")
    for i, c in enumerate(K1_CASES):
        s = replace(c, W=PIN_SIZES[(c.W, c.H)][0], H=PIN_SIZES[(c.W, c.H)][1])
        inp = k1_inputs(s)
        args = k1_call(s, inp, 7001 + i)
        a = orc.ssgi_trace(*args[:-1], inp.blue, out_size=args[-1])
        b = R.ssgi_trace(*args[:-1], inp.blue, out_size=args[-1])
        assert a.tobytes() == b.tobytes(), str(c)
    for c in K2_CASES:
        s = replace(c, W=PIN_SIZES[(c.W, c.H)][0], H=PIN_SIZES[(c.W, c.H)][1])
        p, inp_, vel, h0, h1, t0, t1, half = k2_call(s, k2_inputs(s))
        a = orc.temporal_reproject(p, inp_, vel, h0, h1, t0, t1, out_half=half)
        b = R.temporal_reproject(p, inp_, vel, h0, h1, t0, t1, out_half=half)
        for x, y in zip(a, b):
            assert (x is None and y is None) or x.tobytes() == y.tobytes(), str(c)
    refpins.done(R)
