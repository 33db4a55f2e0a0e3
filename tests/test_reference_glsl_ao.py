"""Reduced-resolution AO (AOEffect's resolutionScale) and K6's normal-texture branch (useNormalPass / normalTexture): the oracle
(tests/ao_harness.py) must equal the reference's own shaders BIT FOR BIT.  The reference side is what its shaders computed for the
same calls, stored as digests in tests/golden/reference_pins_ao.json by tests/golden/make_golden_ao.py (which compares the two live).

What the reference does (src/ao/AOEffect.js:126-154, src/ao/AOPass.js:79-83): the AO pass renders to (int)(W * scale) x (int)(H * scale)
with `resolution` = W * scale x H * scale unrounded; it reads the full-size depth plane by uv and rebuilds the normal in depth texels, or
unpacks the RGBA8 NEAREST view-space normal texture.  The denoiser stays at full size and its first pass samples the AO target LINEAR;
with no denoise iteration the compose samples the AO target itself LINEAR."""
import numpy as np

import ao_harness as ao
import chain_harness as ch

# (width, height, resolutionScale): 66 x 37 at 0.5 is a 33 x 18 target with resolution (33, 18.5)
CASES = [(64, 36, 1.0), (64, 36, 0.75), (64, 36, 0.5), (66, 37, 0.5)]


def run_cases(m) -> list:
    """every case with and without a normal plane: K6 on the AO target, the 2-pass full-size AO denoise from it, ao_compose of the
    denoised plane (iterations > 0) and of the AO target itself (iterations == 0).  m: ao_harness.oracle or the reference"""
    outs = []
    for W, H, scale in CASES:
        inp = ch.make_inputs(W, H, 2)
        f1 = inp.frames[1]
        (tw, th), res = ao.ao_target_size(W, H, scale)
        hp = ao.hbao_params(f1["cam"], 5151)
        z = np.zeros((th, tw, 4), np.float16)
        for normal in (None, ao.view_normal_plane(W, H, 1, f1["cam"])):
            a = m.hbao(hp, f1["depth"], inp.blue, z, out_size=(tw, th), normal=normal, resolution=res)
            assert a.shape == (th, tw, 4) and float(a[..., 3].astype(np.float32).min()) < 0.99  # not an empty plane
            dn = ch.ao_denoise(m, f1, inp.blue, a)
            assert dn[1].shape == (H, W, 4)
            cp = ch.ao_compose_params()
            outs += [a, *dn, m.ao_compose(cp, f1["depth"], dn[1], f1["direct"]), m.ao_compose(cp, f1["depth"], a, f1["direct"])]
    return outs


def test_scaled_ao_and_normal_texture_oracle_equals_reference_shaders():
    ao.check_pins("ao_scaled", run_cases(ao.oracle))


def test_scale_one_without_a_normal_plane_is_the_existing_oracle():
    """at resolutionScale 1 with depth-rebuilt normals the extended oracle computes exactly what tests/orc.py's K6 / K3 / K7 compute"""
    import orc

    inp = ch.make_inputs(64, 36, 2)
    f1 = inp.frames[1]
    hp = ao.hbao_params(f1["cam"], 5151)
    z = np.zeros((36, 64, 4), np.float16)
    a, b = ao.oracle.hbao(hp, f1["depth"], inp.blue, z), orc.hbao(hp, f1["depth"], inp.blue, z)
    assert a.tobytes() == b.tobytes()
    for x, y in zip(ch.ao_denoise(ao.oracle, f1, inp.blue, a), ch.ao_denoise(orc, f1, inp.blue, b)):
        assert x.tobytes() == y.tobytes()
    cp = ch.ao_compose_params()
    assert ao.oracle.ao_compose(cp, f1["depth"], a, f1["direct"]).tobytes() == orc.ao_compose(cp, f1["depth"], b, f1["direct"]).tobytes()


def test_normal_texture_changes_the_result():
    """the normal-texture branch is taken: quantised normals give AO that differs from the depth-rebuilt normals somewhere, while both
    describe the same scene (most foreground normals agree)"""
    W, H = 64, 36
    inp = ch.make_inputs(W, H, 2)
    f1 = inp.frames[1]
    hp = ao.hbao_params(f1["cam"], 5151)
    z = np.zeros((H, W, 4), np.float16)
    a = ao.oracle.hbao(hp, f1["depth"], inp.blue, z)
    b = ao.oracle.hbao(hp, f1["depth"], inp.blue, z, normal=ao.view_normal_plane(W, H, 1, f1["cam"]))
    assert a.tobytes() != b.tobytes()
    fg = f1["depth"] < 1.0
    dot = (a[..., :3].astype(np.float32) * b[..., :3].astype(np.float32)).sum(-1)
    assert float(np.mean(dot[fg] > 0.99)) > 0.8
