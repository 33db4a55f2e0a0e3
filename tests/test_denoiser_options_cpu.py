"""The Poisson denoiser's option space on the CPU: the oracle against the reference's own shaders (tests/refpins.py) at radii, frame
shapes and weights the default options never reach.  tests/test_gpu_denoiser_options.py holds the CUDA kernels to the oracle at the same
points, so the kernels are held to the reference there.

The weight sets: the reference demo's (example/main.js:363-383), all zero, and large (normalPhi 100, lumaPhi 50), where most tap weights
fall under the shader's `w < 0.0001` cutoff.  normalPhi, roughnessPhi and specularPhi differ from each other in the demo and large sets,
so a kernel that read the wrong one of the three gives different bytes."""
import numpy as np

import chain_harness as ch
import orc
import refpins
from realism_effects_b200 import abi

PHIS = {  # (phi, luma_phi, depth_phi, normal_phi, roughness_phi, specular_phi)
    "demo": (0.875, 20.651999999999997, 23.37, 26.087, 18.477999999999998, 7.099999999999999),
    "zero": (0.0, 0.0, 0.0, 0.0, 0.0, 0.0),
    "large": (0.5, 50.0, 10.0, 100.0, 80.0, 60.0),
}


def opts(phis: str, radius: float, **kw) -> ch.Opts:
    phi, luma, depth, normal, rough, spec = PHIS[phis]
    return ch.Opts(radius=float(radius), phi=phi, luma_phi=luma, depth_phi=depth, normal_phi=normal, roughness_phi=rough, specular_phi=spec, **kw)


def velocity_layout_params(o: ch.Opts, index: int) -> abi.PoissonParams:
    """the AO denoiser's form: one plane, normals and depth from the velocity-layout plane (no GBUFFER_TEXTURE), LINEAR fp16 input"""
    p = ch.poisson_params(o, index, False)
    p.texture_count, p.gbuffer_texture, p.input_linear = 1, 0, 1
    p.is_texture_specular[:] = [0, 0]
    return p


def gi_planes(rng, H: int, W: int):
    """two fp32 GI planes like the temporal pass writes them: colours in [0, 4), the age (frames accumulated) in alpha"""
    out = []
    for _ in range(2):
        a = rng.uniform(0.0, 4.0, (H, W, 4)).astype(np.float32)
        a[..., 3] = rng.integers(0, 40, (H, W)).astype(np.float32)
        out.append(a)
    return out


def denoise_and_compose(m, o: ch.Opts, fr: dict, blue, gi, prev16, prev_composed, index: int):
    """pass 0 (NEAREST fp32 in), pass 1 (LINEAR fp16 in), the compose, and one 1-plane velocity-layout pass; `m` runs the passes"""
    a0, a1 = m.poisson_denoise(ch.poisson_params(o, index, True), fr["depth"], fr["gbuffer"], gi[0], gi[1], blue, prev16[0], prev16[1])
    b0, b1 = m.poisson_denoise(ch.poisson_params(o, index + 1, False), fr["depth"], fr["gbuffer"], a0, a1, blue, prev16[1], prev16[0])
    comp = m.gi_compose(ch.compose_params(abi.make_camera(fr["cam"])), fr["depth"], fr["gbuffer"], b0, b1, prev_composed)
    v, _ = m.poisson_denoise(velocity_layout_params(o, index + 2), fr["depth"], fr["velocity"], a0, None, blue, prev16[0], None)
    return a0, a1, b0, b1, comp, v


def test_oracle_equals_reference_shaders_denoiser_option_space():
    """radius 0, 11, 14, 20, 32 at landscape, portrait and square sizes, with each weight set: every output of the Poisson passes in both
    forms and of the compose, bit for bit"""
    R = refpins.ref("denoiser_option_space")
    rng = np.random.default_rng(20261016)
    for W, H in ((48, 28), (28, 48), (36, 36)):
        inp = ch.make_inputs(W, H, 1)
        fr = inp.frames[0]
        assert 0.0 < (fr["depth"] == 1.0).mean() < 1.0  # discarded background next to shaded pixels
        for radius in (0, 11, 14, 20, 32):
            gi = gi_planes(rng, H, W)
            prev16 = [rng.uniform(0.0, 2.0, (H, W, 4)).astype(np.float16) for _ in range(2)]
            prev_composed = rng.uniform(0.0, 2.0, (H, W, 4)).astype(np.float32)
            index = 1000 * radius + W
            outs = set()
            for phis in PHIS:
                o = opts(phis, radius)
                a = denoise_and_compose(orc, o, fr, inp.blue, gi, prev16, prev_composed, index)
                b = denoise_and_compose(R, o, fr, inp.blue, gi, prev16, prev_composed, index)
                for x, y in zip(a, b):
                    assert x.tobytes() == y.tobytes(), (W, H, radius, phis)
                outs.add(a[2].tobytes())
            assert len(outs) == len(PHIS), (W, H, radius)  # same inputs, different weights: different bytes
    refpins.done(R)
