"""The Poisson denoiser (K3, with K4 fused into its last pass) across the options its code paths depend on: the radius, the frame's
aspect ratio and the weights.  One case grid serves every test here.

* The per-pass kernels (rfx_poisson_denoise_launch, fast_math on and off) against the oracle, in both denoiser forms.
* The fast chain's own K3 + K4 kernels (cpoisson_kernel, cpoisson_tma_kernel, the fused compose) against the oracle pass group by pass
  group: the oracle runs the frame's Poisson passes and the compose on the chain's downloaded temporal planes, so K1 / K2 add no drift.
* The TMA-staged passes against the plain ones, byte for byte.  Where the staged tiles do not fit (a box dimension over 256 elements,
  or two tiles over the kernel's shared memory), the plain path must run.
* Row-sharded groups at radius 11, and one process rendering on two devices.

The oracle equals the reference's shaders at these radii, shapes and weights (tests/test_denoiser_options_cpu.py)."""
from __future__ import annotations

import math
import os
from dataclasses import dataclass

import numpy as np
import pytest
import torch

import chain_harness as ch
import orc
from realism_effects_b200 import abi
from test_denoiser_options_cpu import PHIS, opts, velocity_layout_params

PER_PASS_BAR = 1e-4  # fraction of pixels allowed outside 1e-3 relative (the bar of tests/test_gpu_passes.py)

SIZES_RADII = [
    ((200, 120), (0, 1, 3, 11, 32)),           # at 32 the TMA box is refused
    ((120, 200), (3, 11, 13, 14, 21, 22, 32)),  # 13 just fits; 14..21 are too big for the shared memory; from 22 the box is refused
    ((192, 192), (18, 19, 20, 22)),            # 18 fits at 102 144 B, just under the cap
    ((80, 320), (11,)), ((320, 80), (11,)),    # extreme aspect ratios
    ((40, 24), (11,)),                         # no interior block at all
    ((203, 117), (11,)),                       # odd size
]
ITERATIONS = (1, 3, 5)


@dataclass(frozen=True)
class Case:
    W: int
    H: int
    radius: int
    phis: str
    iterations: int

    def __str__(self):
        return f"{self.W}x{self.H}-r{self.radius}-{self.phis}-it{self.iterations}"


def _grid() -> list:
    cases = []
    for (W, H), radii in SIZES_RADII:
        for r in radii:
            for j, phis in enumerate(PHIS):  # every (size, radius) runs each iteration count once, each with other weights
                cases.append(Case(W, H, r, phis, ITERATIONS[(j + r) % len(ITERATIONS)]))
    return cases + [Case(200, 120, 3, "demo", 0), Case(120, 200, 14, "large", 0)]  # no Poisson pass: the stand-alone compose


CASES = _grid()


def k3_path(W: int, H: int, radius: float) -> tuple:
    """which kernel the fast chain's LINEAR Poisson passes take: "tma", "box refused" (a TMA box dimension over 256 elements) or
    "too big" (the two staged tiles over the 100 KB of shared memory the kernel is given); and whether any block is interior (stages
    its tile).  Mirrors chain_render_fast / cpoisson_tma_fits / cpoisson_tma_kernel, in the host's float32 arithmetic."""
    r, w, h = np.float32(radius), np.float32(W), np.float32(H)
    reach_x = int(math.ceil(r * max(np.float32(1.0), w / h))) + 2
    reach_y = int(math.ceil(r * max(np.float32(1.0), h / w))) + 2
    box_w, box_h = (16 + 2 * reach_x) | 1, 16 + 2 * reach_y
    tile = box_w * box_h * 16
    if box_w * 4 > 256 or box_h > 256:
        path = "box refused"
    elif ((tile + 127) & ~127) + tile > 100 * 1024:
        path = "too big"
    else:
        path = "tma"
    interior = any(bx0 - reach_x >= 0 and bx0 - reach_x + box_w - 1 <= W - 1 and by0 - reach_y >= 0 and by0 + 15 + reach_y <= H - 1
                   for by0 in range(0, H, 16) for bx0 in range(0, W, 16))
    return path, interior


def test_case_grid_covers_every_k3_path():
    """(CPU) the grid reaches all three paths, TMA with and without interior blocks, and every iteration count"""
    paths = {c: k3_path(c.W, c.H, c.radius) for c in CASES}
    assert {p for p, _ in paths.values()} == {"tma", "box refused", "too big"}
    assert any(i for p, i in paths.values() if p == "tma") and any(not i for p, i in paths.values() if p == "tma")
    assert {c.iterations for c in CASES} == {0, 1, 3, 5}
    assert k3_path(120, 200, 13) == ("tma", True) and k3_path(192, 192, 18) == ("tma", True)
    assert [k3_path(120, 200, r)[0] for r in (14, 21, 22)] == ["too big", "too big", "box refused"]
    assert [k3_path(192, 192, r)[0] for r in (19, 20, 22)] == ["too big", "too big", "box refused"]
    assert k3_path(3840, 2160, 3) == ("tma", True)  # the benchmarked 4K frame keeps the staged path
    assert k3_path(160, 400, 11)[0] == "too big" and k3_path(320, 304, 11)[0] == "tma"  # the group cases below


# ---- GPU -------------------------------------------------------------------------------------------------------------------------------------
_inputs: dict = {}
_runs: dict = {}


def inputs(W: int, H: int, frames: int = 3) -> ch.Inputs:
    if (W, H, frames) not in _inputs:
        _inputs[(W, H, frames)] = ch.make_inputs(W, H, frames)
    return _inputs[(W, H, frames)]


@pytest.fixture(scope="module")
def ctxs(built):
    """contexts with the TMA-staged Poisson passes on ("tma") and off ("plain"), and one for the per-pass kernels ("pass")"""
    from realism_effects_b200 import engine

    inp = inputs(200, 120)
    out, old = {}, os.environ.get("RFX_K3_TMA")
    try:
        for name, tma in (("tma", "1"), ("plain", "0"), ("pass", "1")):
            os.environ["RFX_K3_TMA"] = tma  # read when the context is created
            c = engine.Context(0, inp.blue)
            c.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
            out[name] = c
    finally:
        if old is None:
            os.environ.pop("RFX_K3_TMA", None)
        else:
            os.environ["RFX_K3_TMA"] = old
    yield out
    _runs.clear()
    for c in out.values():
        c.close()


def chain_run(ctxs, which: str, case: Case) -> list:
    """3 frames of the fast chain; per frame its outputs 0 (composed) and 2..5 (tr0, tr1, dn0, dn1)"""
    from realism_effects_b200 import engine

    key = (which, case)
    if key not in _runs:
        ctx, inp = ctxs[which], inputs(case.W, case.H)
        chain = engine.SsgiChain(ctx, ch.chain_options(inp, opts(case.phis, case.radius, denoise_iterations=case.iterations)))
        try:
            out = []
            for fr in inp.frames:
                planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
                chain.render(abi.make_camera(fr["cam"]), *planes, fr["cam"]["position"], fr["moved"])
                out.append({w: chain.download(w) for w in (0, 2, 3, 4, 5)})
                for p in planes:
                    p.free()
        finally:
            chain.close()
        _runs[key] = out
    return _runs[key]


def check(name, want, got, bar=PER_PASS_BAR):
    c = ch.compare(want, got)
    print(f"{name}: bad={c['frac_bad']:.2e} max_rel_ok={c['max_rel_ok']:.1e} bit_equal={c['bit_equal']:.4f}")
    assert c["frac_bad"] <= bar, (name, c)
    return c


PASS_CASES = [c for c in CASES if c.iterations > 0]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PASS_CASES, ids=str)
def test_per_pass_poisson_kernels_match_the_oracle(ctxs, case):
    """ctx.poisson_denoise, fast_math on and off: 2 planes with the G-buffer (pass 0: fp32 NEAREST in; pass >= 1: fp16 LINEAR in) and the
    1-plane velocity-layout form; on frame 1 of the chain's own planes, into targets holding frame 0's texels (kept where discarded)"""
    ctx, inp = ctxs["pass"], inputs(case.W, case.H)
    run = chain_run(ctxs, "plain", case)
    fr, f0, f1 = inp.frames[1], run[0], run[1]
    o = opts(case.phis, case.radius)
    calls = [
        ("pass 0", ch.poisson_params(o, 777, True), fr["gbuffer"], (f1[2], f1[3]), (f0[4], f0[5])),
        ("pass 1", ch.poisson_params(o, 778, False), fr["gbuffer"], (f1[4], f1[5]), (f0[4], f0[5])),
        ("1-plane", velocity_layout_params(o, 779), fr["velocity"], (f1[4], None), (f0[4], None)),
    ]
    up = lambda a: None if a is None else ctx.upload(a)  # noqa: E731
    d = ctx.upload(fr["depth"])
    try:
        for name, p, nsrc, ins, prevs in calls:
            want = orc.poisson_denoise(p, fr["depth"], nsrc, ins[0], ins[1], inp.blue, prevs[0], prevs[1])
            for fast in (True, False):
                ctx.set_fast_math(fast)
                outs = [up(x) for x in prevs]
                ctx.poisson_denoise(p, d, ctx.upload(nsrc), up(ins[0]), up(ins[1]), outs[0], outs[1])
                for k in range(2 if ins[1] is not None else 1):
                    check(f"{case} {name} plane {k} fast={fast}", want[k], outs[k].download())
    finally:
        ctx.set_fast_math(True)


# Bars of the fast chain's pass groups by denoiseIterations, against the worst plane measured over the grid on an H100 80GB HBM3
# (700 W): 0 passes 0; 1 iteration 3.5e-4; 3 iterations 7.9e-4; 5 iterations 9.2e-4 apart from the case below.  Each pass alone is
# within the per-pass bar (0 pixels out, test above); what grows with the passes is that a pass's output is the next one's input, so
# a last-bit difference of the fast kernels' SFU lg2 / ex2 from the oracle's libm that flips one fp16 rounding is carried and can
# flip the next.  (Up to 9 pixels of dn0 on 80x320 at radius 11 with all weights 0 are not traced to the pixel.  Frame 0's `composed`
# on 120x200 had 4 pixels 1.2e-3 off in 15 cases while c_compose formed the perspective viewZ with a reciprocal; with one division, as
# perspectiveDepthToViewZ, those 15 cases have none, H100 80GB HBM3, 700 W.)
CHAIN_BAR = {0: PER_PASS_BAR, 1: 5e-4, 3: 1e-3, 5: 1e-3}
# Measured 1.37e-3 (33 pixels of dn1, frame 0).  18 of them are flat pixels whose every tap weight is cut (w < 0.0001) by the large
# weights, so each pass writes fp16(1.0003 * c) (the centre's factor, poisson_denoise.frag); near c = 1.6276 that product is half an fp16
# ulp above c, the oracle rounds down every pass and the fast kernel up, 1 ulp per pass: 9 ulps (0.55 %) after 10 passes.
TIE_DRIFT = {Case(120, 200, 3, "large", 5)}
CHAIN_CASES = [pytest.param(c, marks=pytest.mark.xfail(strict=True, reason="fp16 rounding ties compound over 10 passes")) if c in TIE_DRIFT else c
               for c in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CHAIN_CASES, ids=str)
def test_fast_chain_poisson_and_compose_match_the_oracle(ctxs, case):
    """two frames of the fast chain: the oracle runs each frame's Poisson passes (blue-noise indices continuing across frames like the
    chain's) and the compose on the chain's downloaded tr0 / tr1, with last frame's downloaded dn0 / dn1 and composed as the targets'
    kept texels and its own A target; it must give this frame's outputs 4, 5 and 0"""
    inp = inputs(case.W, case.H)
    run = chain_run(ctxs, "tma", case)
    o = opts(case.phis, case.radius, denoise_iterations=case.iterations)
    H, W = inp.height, inp.width
    z16 = np.zeros((H, W, 4), np.float16)
    dnA, prev_dn, prev_comp, bn = [z16, z16], [z16, z16], np.zeros((H, W, 4), np.float32), 0
    for t in range(2):
        fr, got = inp.frames[t], run[t]
        tr, dnB = [got[2], got[3]], list(prev_dn)
        for i in range(2 * case.iterations):
            horizontal = i % 2 == 0
            src = tr if i == 0 else (dnB if horizontal else dnA)
            dst = dnA if horizontal else dnB
            bn = ch.next_blue(o.blue_noise_start, bn)
            out = list(orc.poisson_denoise(ch.poisson_params(o, bn, i == 0), fr["depth"], fr["gbuffer"], src[0], src[1], inp.blue, dst[0], dst[1]))
            if horizontal:
                dnA = out
            else:
                dnB = out
        comp = orc.gi_compose(ch.compose_params(abi.make_camera(fr["cam"])), fr["depth"], fr["gbuffer"], dnB[0], dnB[1], prev_comp)
        bar = CHAIN_BAR[case.iterations]
        check(f"{case} f{t} dn0", dnB[0], got[4], bar)
        check(f"{case} f{t} dn1", dnB[1], got[5], bar)
        check(f"{case} f{t} composed", comp, got[0], bar)
        prev_dn, prev_comp = [got[4], got[5]], got[0]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=str)
def test_tma_staged_and_plain_poisson_passes_write_the_same_bytes(ctxs, case):
    """RFX_K3_TMA=1 against RFX_K3_TMA=0 over 3 frames, outputs 0 and 2..5"""
    a, b = chain_run(ctxs, "tma", case), chain_run(ctxs, "plain", case)
    for t in range(3):
        for w in (0, 2, 3, 4, 5):
            assert a[t][w].tobytes() == b[t][w].tobytes(), (str(case), k3_path(case.W, case.H, case.radius), t, w)


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(160, 400), (320, 304)])
@pytest.mark.parametrize("mode", [abi.MODE_SSGI, abi.MODE_SSR], ids=["fast-chain", "ssr-per-pass-chain"])
def test_row_sharded_group_at_radius_11_equals_one_chain(built, mode, W, H):
    """an in-process group of 3 bands (the fast chain in SSGI mode, the per-pass chain in SSR mode with denoiseMode "full") at radius 11
    with the demo's weights; 160x400 is too big for the staged tiles, 320x304 takes them.  Borders move once; every output equals one
    chain byte for byte."""
    from realism_effects_b200 import engine, parallel

    world = 3
    o = opts("demo", 11, mode=mode, denoise_iterations=2)
    inp = ch.make_inputs(W, H, 4, fov=75.0)  # the sky's silhouette crosses the band borders
    outputs = (0, 1, 2, 3, 4, 5) if mode == abi.MODE_SSGI else (0, 1, 2, 4)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, o)
        single = engine.SsgiChain(ctx, copt)
        grp = parallel.InProcessGroup(ctx, copt, world)
        b = list(grp.bounds)
        for t, fr in enumerate(inp.frames):
            if t == 2:
                grp.set_bounds([0] + [x + 16 for x in b[1:-1]] + [H])
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            cam = abi.make_camera(fr["cam"])
            single.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            grp.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            for which in outputs:
                a, g = single.download(which), grp.download(which)
                if a.tobytes() != g.tobytes():
                    rows = np.nonzero((a.view(np.uint8).reshape(H, -1) != g.view(np.uint8).reshape(H, -1)).any(1))[0]
                    raise AssertionError(f"frame {t} output {which}: rows {rows[0]}..{rows[-1]} differ ({len(rows)} rows); bounds {grp._last_bounds}")
            for p in planes:
                p.free()
        grp.close()
        single.close()
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_devices_in_one_process_render_the_same_bytes(built):
    """contexts on devices 0 and 1 of one process, the fast chain at radius 11 (staged tiles of ~80 KB: over the 48 KB a kernel gets without
    raising its shared-memory attribute, which is set per device) on each"""
    from realism_effects_b200 import engine

    case = Case(200, 120, 11, "demo", 2)
    assert k3_path(case.W, case.H, case.radius) == ("tma", True)
    inp = inputs(case.W, case.H)
    o = opts(case.phis, case.radius, denoise_iterations=case.iterations)
    ctx = [engine.Context(d, inp.blue) for d in (0, 1)]
    try:
        chains = []
        for c in ctx:
            c.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
            chains.append(engine.SsgiChain(c, ch.chain_options(inp, o)))
        for t, fr in enumerate(inp.frames):
            got = []
            for c, chain in zip(ctx, chains):
                planes = [c.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
                chain.render(abi.make_camera(fr["cam"]), *planes, fr["cam"]["position"], fr["moved"])
                got.append({w: chain.download(w).tobytes() for w in (0, 2, 3, 4, 5)})
                for p in planes:
                    p.free()
            assert got[0] == got[1], t
        for chain in chains:
            chain.close()
    finally:
        for c in ctx:
            c.close()
