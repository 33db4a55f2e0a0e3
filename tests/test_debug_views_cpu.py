"""CPU tests of the debug views (SSGIEffect's `outputTexture`, src/ssgi/SSGIEffect.js:228-251): the oracle's GBufferDebugPass and K5
debug branch held bit for bit to the reference's own shaders (through tests/golden/reference_pins_debug.json, and directly where the
reference checkout is present), the setter's rules on the host side, and the ABI mirrors of include/rfx.h."""
import re

import numpy as np
import pytest

import debug_views as D
from realism_effects_b200 import abi, effects

RFX_H = D.os.path.join(D.ROOT, "include", "rfx.h")


@pytest.mark.parametrize("size", D.GB_SIZES)
def test_gbuffer_debug_oracle_matches_reference_pins(size):
    W, H = size
    outs = D.pin_cases(D.oracle)
    D.check_pins(f"gbuffer_debug_{W}x{H}", outs[f"gbuffer_debug_{W}x{H}"])


def test_gbuffer_debug_emissive_every_exponent_matches_reference_pins():
    """every exponent byte of decodeRGBE8 (256 values of fExp) through the emissive mode"""
    D.check_pins("gbuffer_debug_rgbe", [D.oracle.gbuffer_debug(5, D.rgbe_gbuffer())])


@pytest.mark.parametrize("size", D.K5_SIZES)
def test_k5_debug_oracle_matches_reference_pins(size):
    W, H = size
    D.check_pins(f"k5_debug_{W}x{H}", [D.oracle.ssgi_compose_debug(v, (W, H)) for _, v in D.k5_views(W, H)])


@pytest.mark.skipif(not D.reference_available(), reason="needs the reference checkout")
def test_oracle_equals_reference_shaders_directly():
    for (tag, a), (_, b) in zip(D.pin_cases(D.oracle).items(), D.pin_cases(D.reference).items()):
        for i, (x, y) in enumerate(zip(a, b)):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), (tag, i)


def test_gbuffer_debug_masks_zero_albedo_bits_and_unknown_mode_is_emissive():
    """the pass's unbound depthTexture reads gBuffer.r: the cleared texel and both transparent-black blocks are vec4(0); an unknown mode
    (-1) takes the shader's else branch"""
    fr = D.debug_frame(61, 35)
    g = fr["gbuffer"]
    zero = g[..., 0] == 0.0
    assert zero.any() and (g[..., 0].view(np.uint32) == 0x80000000).any()
    for mode in range(6):
        o = D.oracle.gbuffer_debug(mode, g)
        assert (o[zero] == 0).all() and (o[~zero][:, 3] == 1).all()
    assert np.array_equal(D.oracle.gbuffer_debug(-1, g), D.oracle.gbuffer_debug(5, g))
    assert np.array_equal(D.oracle.gbuffer_debug(17, g), D.oracle.gbuffer_debug(5, g))


def test_k5_debug_linear_fetch_at_odd_size_is_not_a_copy():
    """dnB is sampled LINEAR at the pixel centre: ((x+.5)/W)*W-.5 is not always x, so somewhere the result is not the texel itself"""
    W, H = 203, 117
    v = dict(D.k5_views(W, H))["dnB"]
    got = D.oracle.ssgi_compose_debug(v, (W, H))
    assert not np.array_equal(got.view(np.uint16), v.view(np.uint16))
    assert np.abs(got.astype(np.float64) - v.astype(np.float64)).max() < 0.05


def test_k5_debug_depth_reads_d001():
    W, H = 64, 36
    d = dict(D.k5_views(W, H))["depth"]
    got = D.oracle.ssgi_compose_debug(d, (W, H)).astype(np.float32)
    assert np.array_equal(got[..., 0], d.astype(np.float16).astype(np.float32))
    assert (got[..., 1:3] == 0).all() and (got[..., 3] == 1).all()


def _defines(text):
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (RFX_DEBUG_VIEW_\w+) \(?(-?\d+)\)?", text)}


def test_abi_debug_view_mirror():
    with open(RFX_H, encoding="utf-8") as f:
        d = _defines(f.read())
    assert d == {"RFX_DEBUG_VIEW_NONE": abi.DEBUG_VIEW_NONE, "RFX_DEBUG_VIEW_OUTPUT": abi.DEBUG_VIEW_OUTPUT, "RFX_DEBUG_VIEW_DEPTH": abi.DEBUG_VIEW_DEPTH,
                 "RFX_DEBUG_VIEW_VELOCITY": abi.DEBUG_VIEW_VELOCITY, "RFX_DEBUG_VIEW_GBUFFER": abi.DEBUG_VIEW_GBUFFER,
                 "RFX_DEBUG_VIEW_GBUFFER_CHANNEL": abi.DEBUG_VIEW_GBUFFER_CHANNEL}
    assert abi.GBUFFER_DEBUG_MODES == ["diffuse", "alpha", "normal", "roughness", "metalness", "emissive"]
    for n in ("rfx_gbuffer_debug_launch", "rfx_ssgi_chain_set_debug_view"):
        assert n in abi.EXPORTS


def test_gbuffer_debug_launch_declaration_matches_binding():
    with open(RFX_H, encoding="utf-8") as f:
        t = f.read()
    m = re.search(r"rfx_status rfx_gbuffer_debug_launch\(([^)]*)\)", t)
    assert m and len(m.group(1).split(",")) == 7
    m = re.search(r"rfx_status rfx_ssgi_chain_set_debug_view\(([^)]*)\)", t)
    assert m and "int32_t view" in m.group(1)


def test_debug_view_rule_of_the_setter():
    """_debug_state: the reference setter's outcome for each kind of value, without a GPU (SSGIEffect.js:228-251)"""
    assert effects._debug_state("normal") == ("gbuffer", 2)
    assert effects._debug_state("diffuse") == ("gbuffer", 0)
    assert effects._debug_state("bogus") == ("gbuffer", -1)
    assert effects._debug_state(abi.Plane()) == ("texture", None)
    assert effects._debug_state(None) is None and effects._debug_state("") is None
