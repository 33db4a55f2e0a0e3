"""The fast chain's K1 plane (chain output 1, ssgi_fast_kernel) byte for byte against SHA-256 digests of the same seeded inputs.

A restructured march that keeps each ray's operations (which lane marches a ray, in what order the warp's rays run; DESIGN.md §4)
must keep every byte of the plane, so any difference here is a bug, not rounding.  The digests were taken from the per-pixel march.
The cases reach partial warps and blocks, SSR mode (one ray per pixel), steps = 1 (no step tested) and refineSteps = 0, missed rays,
a non-sparse (orthographic) projection and a 3-band in-process group (the PEER read of last frame's `composed`).
Two frames each: the second reads the first one's `composed`."""
from __future__ import annotations

import hashlib

import pytest

import chain_harness as ch
from realism_effects_b200 import abi

FRAMES = 2

# case: (width, height, Opts overrides, make_inputs overrides, group members)
CASES = {
    "bench_4k": (3840, 2160, dict(denoise_iterations=2), dict(reference_env=True, device="cuda"), 1),
    "203x117": (203, 117, {}, {}, 1),
    "13x9": (13, 9, {}, {}, 1),
    "ssr": (203, 117, dict(mode=abi.MODE_SSR), {}, 1),
    "steps1_refine0": (203, 117, dict(steps=1, refine_steps=0), {}, 1),
    "steps33_refine0": (203, 117, dict(steps=33, refine_steps=0), {}, 1),
    "missed_rays": (203, 117, dict(missed_rays=True), {}, 1),
    "orthographic": (203, 117, {}, dict(orthographic=True), 1),
    "group3": (320, 304, {}, dict(fov=75.0), 3),
}

DIGESTS = {
    "bench_4k": "e16d626081c5b138fc7b0801491e63e56edd58bcf74ed7cbdba18fafada87c4c",
    "203x117": "0095b2880aa4c3bed12451aca2c028fd2b20142d899c45f9e0cd0480b30ffdad",
    "13x9": "903bdf649bd6d4b0ad633163f9e794badea39ef8d538fca1f7e3a5e18c18ece7",
    "ssr": "adc4cbcbc722da262321b45ba536d1612320f6dff8cef30f6c44b8371f870df4",
    "steps1_refine0": "5427d46151b4d7044ef80d9506383ecc6652f67a8a6bd4adb5d552cd01ade691",
    "steps33_refine0": "b1d169f2e4a0dcbd2b9bcf19672d1e1d2d6499459885e2f80836de9bbb12c6d9",
    "missed_rays": "1b8c71e256978112e31d790e7457f240951f29295be334ae99ff5ae4b420b123",
    "orthographic": "38757dc845f2aa8b24906b436fa830e3e34b1386112ae1c88f657f5c4f6b3b0f",
    "group3": "b7632fe1ca3bb6d65b0df21fdd35b84022d029420ae667b8e5a7cb08f78d2e73",
}


def k1_digest(name: str) -> str:
    """SHA-256 of the K1 plane of every frame of case `name`, in frame order"""
    from realism_effects_b200 import engine, parallel

    W, H, opts, inp_kw, world = CASES[name]
    o = ch.Opts(**opts)
    inp = ch.make_inputs(W, H, FRAMES, **inp_kw)
    ctx = engine.Context(0, inp.blue)
    h = hashlib.sha256()
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, o)
        chain = parallel.InProcessGroup(ctx, copt, world) if world > 1 else engine.SsgiChain(ctx, copt)
        for fr in inp.frames:
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            chain.render(abi.make_camera(fr["cam"]), *planes, fr["cam"]["position"], fr["moved"])
            h.update(chain.download(1).tobytes())
            for p in planes:
                p.free()
        chain.close()
    finally:
        ctx.close()
    return h.hexdigest()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_k1_plane_keeps_its_bytes(built, name):
    assert k1_digest(name) == DIGESTS[name]
