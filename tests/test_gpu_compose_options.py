"""The GI compose (K4) and the SSGI compose (K5) across their option space.  The case grids and what each case reaches are in
tests/test_compose_options_cpu.py, which also holds the oracle to the reference's shaders at the same points.

* The per-pass K4 (ctx.gi_compose), fast math on and off: the exact variant bit-equal to the oracle (DESIGN.md §2), the fast variant
  to the per-pass bar; discarded pixels keep the target's bytes; two row-range launches split at an odd row write the bytes of one.
* The per-pass K5 (ctx.ssgi_compose) over the K5 grid: bit-equal to the oracle, and the same row-range check.
* The fast chain's own K4 (c_compose in ccompose_kernel, cpoisson_kernel and cpoisson_tma_kernel) over 3 frames on the material-edge
  G-buffer, at 200x120 and on 3840x16 strips: each frame's output 0 against the oracle's compose of the chain's own outputs 4 and 5
  (dn0, dn1) over its last output 0, so no Poisson drift is carried in.
The chain's TRAA tail runs with each K5 grid point as its compose options in tests/test_gpu_traa_tail.py."""
from __future__ import annotations

import os

import numpy as np
import pytest

import chain_harness as ch
import orc
from realism_effects_b200 import abi
from test_compose_options_cpu import CHAIN_CASES, K4_CASES, K5_CASES, ChainCase, K4Case, K5Case, chain_inputs, k4_call, k5_call

PER_PASS_BAR = 1e-4  # fraction of pixels allowed outside 1e-3 relative (the bar of tests/test_gpu_passes.py)


@pytest.fixture(scope="module")
def ctxs(built):
    """contexts with the TMA-staged Poisson passes on ("tma") and off ("plain"); the per-pass tests use "tma" """
    from realism_effects_b200 import engine

    inp = chain_inputs(200, 120, "sym")
    out, old = {}, os.environ.get("RFX_K3_TMA")
    try:
        for name, tma in (("tma", "1"), ("plain", "0")):
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
    for c in out.values():
        c.close()


def split_row(H: int) -> int:
    return min((H // 2) | 1, H - 1)


def first_diff(name: str, want: np.ndarray, got: np.ndarray):
    bad = (want.view(np.uint32) != got.view(np.uint32)).reshape(want.shape[0], want.shape[1], -1).any(-1)
    assert not bad.any(), f"{name}: {int(bad.sum())} pixels differ from the oracle, first at (y, x) = {tuple(int(v) for v in np.argwhere(bad)[0])}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", K4_CASES, ids=str)
def test_per_pass_k4_matches_the_oracle(ctxs, case: K4Case):
    ctx = ctxs["tma"]
    p, depth, gb, d, s, prev, scene = k4_call(case)
    want = orc.gi_compose(p, depth, gb, d, s, prev, scene=scene)
    kept = (want.view(np.uint32) == prev.view(np.uint32)).all(-1)
    assert kept.any() and not kept.all()
    up = lambda a: None if a is None else ctx.upload(a)  # noqa: E731
    ins = [up(a) for a in (depth, gb, d, s, scene)]
    H, r = depth.shape[0], split_row(depth.shape[0])
    try:
        for fast in (True, False):
            ctx.set_fast_math(fast)
            whole, split = ctx.upload(prev), ctx.upload(prev)
            ctx.gi_compose(p, *ins[:4], whole, scene=ins[4])
            for rows in ((0, r), (r, H)):
                ctx.gi_compose(p, *ins[:4], split, rows=rows, scene=ins[4])
            got = whole.download()
            assert split.download().tobytes() == got.tobytes(), f"{case} fast={fast}: rows [0, {r}) + [{r}, {H}) differ from one launch"
            assert (got.view(np.uint32)[kept] == prev.view(np.uint32)[kept]).all(), f"{case} fast={fast}: a discarded pixel was written"
            c = ch.compare(want, got)
            print(f"{case} fast={fast}: bad={c['frac_bad']:.2e} n_bad={c['n_bad']} max_rel_ok={c['max_rel_ok']:.1e} bit_equal={c['bit_equal']:.4f}")
            assert c["frac_bad"] <= PER_PASS_BAR, (str(case), fast, c)
            if not fast:
                first_diff(f"{case} exact", want, got)
            whole.free()
            split.free()
    finally:
        ctx.set_fast_math(True)
        for q in ins:
            if q is not None:
                q.free()


@pytest.mark.gpu
@pytest.mark.parametrize("case", K5_CASES, ids=str)
def test_per_pass_k5_matches_the_oracle(ctxs, case: K5Case):
    ctx = ctxs["tma"]
    depth, gi, scene, p = k5_call(case)
    want = orc.ssgi_compose(depth, gi, scene, p)
    ins = [ctx.upload(a) for a in (depth, gi, scene)]
    H, W = depth.shape
    r = split_row(H)
    out, split = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
    try:
        for fast in (True, False):
            ctx.set_fast_math(fast)
            ctx.ssgi_compose(*ins, out, params=p)
            for rows in ((0, r), (r, H)):
                ctx.ssgi_compose(*ins, split, rows=rows, params=p)
            got = out.download()
            assert split.download().tobytes() == got.tobytes(), f"{case} fast={fast}: rows [0, {r}) + [{r}, {H}) differ from one launch"
            bad = (want.view(np.uint16) != got.view(np.uint16)).any(-1)
            assert not bad.any(), f"{case} fast={fast}: {int(bad.sum())} pixels differ from the oracle, first at (y, x) = {tuple(int(v) for v in np.argwhere(bad)[0])}"
    finally:
        ctx.set_fast_math(True)
        for q in ins + [out, split]:
            q.free()


# ---- the fast chain's own K4 ---------------------------------------------------------------------------------------------------------------
# c_compose must form the perspective viewZ with one division, as perspectiveDepthToViewZ does: near d = 1 the denominator cancels,
# and the extra rounding of (n f) * (1 / ((f - n) d - f)) changes the composed colour of 65 pixels (2.7e-3) of frame 0 of the symmetric
# cases here by up to 70 %.
# What remains is c_compose's pixel-centre fetch of dn: it takes the centre texel, where the shader's LINEAR sampler weighs in the
# neighbours by a few ulps of u * W - 0.5.  The literal fetch is not possible in the fused last Poisson pass: the neighbours' dn texels
# are written by other blocks of the same launch.  Measured on an H100 80GB HBM3 (700 W): at 200 x 120 one pixel, (62, 177) of frame 2
# of the orthographic cases; on the 3840 x 16 strips, where those ulps are largest, 3.6e-4 to 8.8e-4 of each frame.  The test shows the
# cause: against the oracle fed the same dn planes as RGBA32F (NEAREST, the centre texel) no pixel of any case is over the bar.
CENTRE_TEXEL = {(str(c), 2): {(62, 177)} for c in CHAIN_CASES if (c.W, c.H, c.camera) == (200, 120, "ortho") and c.iterations > 0}
WIDE_BAR = 1e-3  # the strips, against the LINEAR oracle


@pytest.mark.gpu
@pytest.mark.parametrize("case", CHAIN_CASES, ids=str)
def test_fast_chain_compose_matches_the_oracle(ctxs, case: ChainCase):
    """3 frames of the fast chain (SSGI mode) on the material-edge G-buffer; per frame, output 0 against orc.gi_compose of the chain's
    own outputs 4 and 5 with its last output 0 as the kept texels"""
    from realism_effects_b200 import engine

    ctx = ctxs["tma" if case.tma else "plain"]
    inp = chain_inputs(case.W, case.H, case.camera)
    chain = engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts(denoise_iterations=case.iterations)))
    prev = np.zeros((case.H, case.W, 4), np.float32)
    try:
        for t, fr in enumerate(inp.frames):
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            cam = abi.make_camera(fr["cam"])
            chain.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            got = {w: chain.download(w) for w in (0, 4, 5)}
            for q in planes:
                q.free()
            p = ch.compose_params(cam)
            want = orc.gi_compose(p, fr["depth"], fr["gbuffer"], got[4], got[5], prev)
            centre = orc.gi_compose(p, fr["depth"], fr["gbuffer"], got[4].astype(np.float32), got[5].astype(np.float32), prev)
            cc = ch.compare(centre, got[0])
            assert cc["n_bad"] == 0, (f"{case} f{t} against the centre-texel oracle", cc)
            c = ch.compare(want, got[0])
            print(f"{case} f{t}: bad={c['frac_bad']:.2e} n_bad={c['n_bad']} max_rel_ok={c['max_rel_ok']:.1e} bit_equal={c['bit_equal']:.4f}")
            if case.W > 1000:
                assert c["frac_bad"] <= WIDE_BAR, (f"{case} f{t}", c)
            else:
                A, B = want.astype(np.float64), got[0].astype(np.float64)
                bad = {(int(y), int(x)) for y, x in np.argwhere((np.abs(A - B) > ch.RTOL * np.maximum(np.abs(A), np.abs(B)) + ch.ATOL).any(-1))}
                assert bad <= CENTRE_TEXEL.get((str(case), t), set()), (f"{case} f{t}", c, sorted(bad))
            prev = got[0]
    finally:
        chain.close()
