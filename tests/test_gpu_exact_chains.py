"""The exact SSGI and SSR chains (fast_math off) end to end against the oracle chain, byte for byte.

Every kernel the exact per-pass chain launches (K1, K2, K3, K4 and, in the modes without Poisson passes, the FramebufferTexture copy)
is bit-equal to the oracle on its own (tests/test_gpu_march_options.py, test_gpu_denoiser_options.py, test_gpu_compose_options.py).  So
over several moving frames with history, every plane the chain keeps (the K1 target, the temporal targets, the Poisson targets and
`composed`) must equal the oracle chain's bytes on every frame: in SSGI and SSR mode, in every denoise mode, with 0, 1 and 3 denoise
iterations, at a reduced resolutionScale, with a static camera (the full-accumulate path), an orthographic camera and an odd frame size.
A failure names the first frame, plane and pixel that differ."""
from __future__ import annotations

import pytest

import chain_harness as ch
from realism_effects_b200 import abi

pytestmark = pytest.mark.gpu

SSGI, SSR = abi.MODE_SSGI, abi.MODE_SSR
FULL, FULL_TEMPORAL, TEMPORAL = 0, abi.DENOISE_FULL_TEMPORAL, abi.DENOISE_TEMPORAL

# (id, width, height, frames, make_inputs keywords, Opts keywords)
CASES = [
    ("ssgi-full", 160, 96, 4, {}, dict(mode=SSGI)),
    ("ssgi-full_temporal", 160, 96, 4, {}, dict(mode=SSGI, denoise_mode=FULL_TEMPORAL)),
    ("ssgi-temporal", 160, 96, 4, {}, dict(mode=SSGI, denoise_mode=TEMPORAL)),
    ("ssr-full", 160, 96, 4, {}, dict(mode=SSR)),
    ("ssr-full_temporal", 160, 96, 4, {}, dict(mode=SSR, denoise_mode=FULL_TEMPORAL)),
    ("ssr-temporal", 160, 96, 4, {}, dict(mode=SSR, denoise_mode=TEMPORAL)),
    ("ssgi-it0", 160, 96, 3, {}, dict(mode=SSGI, denoise_iterations=0)),
    ("ssgi-it3", 160, 96, 3, {}, dict(mode=SSGI, denoise_iterations=3)),
    ("ssr-it0", 160, 96, 3, {}, dict(mode=SSR, denoise_iterations=0)),
    ("ssr-it3", 160, 96, 3, {}, dict(mode=SSR, denoise_iterations=3)),
    ("ssgi-scale0.5", 160, 96, 3, {}, dict(mode=SSGI, resolution_scale=0.5)),
    ("ssgi-scale0.75", 160, 96, 3, {}, dict(mode=SSGI, resolution_scale=0.75)),
    ("ssr-scale0.5", 160, 96, 3, {}, dict(mode=SSR, resolution_scale=0.5)),
    ("ssgi-scale0.75-full_temporal", 160, 96, 3, {}, dict(mode=SSGI, resolution_scale=0.75, denoise_mode=FULL_TEMPORAL)),
    ("ssgi-static", 160, 96, 4, dict(static=True), dict(mode=SSGI)),
    ("ssr-static", 160, 96, 4, dict(static=True), dict(mode=SSR)),
    ("ssgi-ortho", 160, 90, 3, dict(orthographic=True), dict(mode=SSGI)),
    ("ssr-ortho", 160, 90, 3, dict(orthographic=True), dict(mode=SSR)),
    ("ssgi-odd-it2", 157, 93, 3, {}, dict(mode=SSGI, denoise_iterations=2)),
    ("ssr-odd", 157, 93, 3, {}, dict(mode=SSR)),
]


def planes_of(o: ch.Opts) -> tuple:
    """the planes the chain keeps in this mode: SSR has one temporal and one Poisson plane; without Poisson passes there are none"""
    tr = ("tr0", "tr1") if o.mode == SSGI else ("tr0",)
    dn = () if o.denoise_mode != FULL else (("dn0", "dn1") if o.mode == SSGI else ("dn0",))
    return ("ssgi", *tr, *dn, "composed")


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_exact_chain_equals_the_oracle_chain_byte_for_byte(built, case):
    name, W, H, frames, inputs_kw, opt_kw = case
    o = ch.Opts(**opt_kw)
    inp = ch.make_inputs(W, H, frames, **inputs_kw)
    planes = planes_of(o)
    ref = ch.run_oracle_chain(inp, o, capture=planes, lean=True)
    got, launches = ch.run_cuda_chain(inp, o, capture=planes, fast_math=False)
    assert launches > 0
    if o.resolution_scale != 1.0:
        assert got[0]["ssgi"].shape[:2] == (int(H * o.resolution_scale), int(W * o.resolution_scale))
    differ = [r for t in range(frames) for k in planes for r in [ch.byte_report(f"{name} frame {t} {k}", ref[t][k], got[t][k])] if r]
    assert not differ, f"{len(differ)} planes differ; first: {differ[0]}"
