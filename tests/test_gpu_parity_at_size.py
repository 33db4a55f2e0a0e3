"""Oracle-vs-CUDA parity at the BASELINE config sizes (VERDICT r1 item 1): C2 1920x1080 (SSGIEffect defaults), C3 3840x2160
(denoiseIterations 2; the workload bench.py times, fast variant, and the exact variant) over 3 frames with history, every
plane of every frame; and C4 (HBAO 4K + 2 single-plane Poisson passes + ao_compose).

The exact variant runs kernels that are each bit-equal to the oracle: every plane of every frame must equal the oracle's byte for byte.
Bars of the fast variant: the fraction of pixels with any channel outside |a-b| <= 1e-3*max(|a|,|b|) + 1e-5 stays below 1e-3 for every
plane of every frame (the residue is 1-fp16-ulp = 9.8e-4 differences at the quantisation points, where the SFU transcendentals differ
from the oracle in the last bits), below 2e-4 outside 4e-3, and K1's own output below 5e-4 (a few rays resolve differently; the rest is
the fed-back history)."""
import os
import sys

import numpy as np
import pytest

import chain_harness as ch
from realism_effects_b200 import abi, engine

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


def _check(res, variant, bar_1e3=1e-3, bar_4e3=2e-4, bar_k1=5e-4):
    d = res["variants"][variant]
    print(res["config"], variant, "worst@1e-3", d["worst_frac_bad_1e3"], "worst@4e-3", d["worst_frac_bad_4e3"])
    for row in d["rows"]:
        assert row["frac_bad_1e3"] <= bar_1e3 and row["frac_bad_4e3"] <= bar_4e3, (res["config"], variant, row)
        if row["plane"] == "ssgi":
            assert row["frac_bad_1e3"] <= bar_k1, (res["config"], variant, row)
    assert d["launches"] > 0


def _check_bytes(res, variant="exact"):
    d = res["variants"][variant]
    bad = [(r["frame"], r["plane"], r["n_differ"], r["first_differ"]) for r in d["rows"] if r["n_differ"]]
    assert not bad, (res["config"], variant, "(frame, plane, pixels that differ, first (y, x))", bad)
    assert d["launches"] > 0


def test_c2_1080p_three_frames_fast_and_exact(built):
    import parity_at_size as pas

    res = pas.run("C2", 3, variants=(True, False))
    _check(res, "fast")
    _check_bytes(res)


def test_c3_4k_three_frames_fast_and_exact(built):
    import parity_at_size as pas

    res = pas.run("C3", 3, variants=(True, False))
    _check(res, "fast")
    _check_bytes(res)


def test_c4_hbao_4k_with_denoise_and_compose(built):
    """K6 (spp form) -> 2 single-plane Poisson passes (velocity-layout normals) -> K7 at 3840x2160 against the oracle, in both variants.
    K6 and K7 are bit-equal in both; the exact K3 is bit-equal, the fast K3 (SFU lg2 / ex2) within 1e-3 on 1e-3 of the pixels, and the
    fast K7, fed the fast K3's plane, as well."""
    import orc

    W, H = 3840, 2160
    inp = ch.make_inputs(W, H, 1)
    fr = inp.frames[0]
    z = np.zeros((H, W, 4), np.float16)
    hp = ch.hbao_params(fr["cam"], 778)
    want_ao = orc.hbao(hp, fr["depth"], inp.blue, z)
    pps, want3, cur = [], [], want_ao
    for i in range(2):
        p = ch.poisson_params(ch.Opts(), 1234568 + i, False)
        p.texture_count, p.gbuffer_texture, p.input_linear = 1, 0, 1
        p.is_texture_specular[:] = [0, 0]
        p.normal_phi, p.depth_phi, p.roughness_phi, p.specular_phi = 3.25, 2.0, 0.0, 0.0
        cur, _ = orc.poisson_denoise(p, fr["depth"], fr["velocity"], cur, None, inp.blue, z, None)
        pps.append(p)
        want3.append(cur)
    want7 = orc.ao_compose(ch.ao_compose_params(), fr["depth"], cur, fr["direct"])
    for fast in (True, False):
        ctx = engine.Context(0, inp.blue)
        try:
            ctx.set_fast_math(fast)
            d, v, dl = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            ao = ctx.upload(z)
            ctx.hbao(hp, d, ao)
            assert not ch.byte_report("K6", want_ao, ao.download()), ch.byte_report(f"K6 fast={fast}", want_ao, ao.download())
            src_g = ao
            for i in range(2):
                dst_g = ctx.upload(z)
                ctx.poisson_denoise(pps[i], d, v, src_g, None, dst_g, None)
                got = dst_g.download()
                if fast:
                    c = ch.compare(want3[i], got)
                    assert c["frac_bad"] <= 1e-3, (f"K3 pass {i}", c)
                else:
                    assert not ch.byte_report("", want3[i], got), ch.byte_report(f"K3 pass {i}", want3[i], got)
                src_g = dst_g
            outp = ctx.alloc(abi.FMT_RGBA16F, W, H)
            ctx.ao_compose(ch.ao_compose_params(), d, src_g, dl, outp)
            got = outp.download()
            if fast:
                c = ch.compare(want7, got)
                assert c["frac_bad"] <= 1e-3, ("K7", c)
            else:
                assert not ch.byte_report("", want7, got), ch.byte_report("K7", want7, got)
        finally:
            ctx.close()
