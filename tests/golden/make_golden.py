"""Mint the golden fixtures from THE REFERENCE'S OWN SHADERS, compiled for the CPU (tests/refglsl.py: the GLSL under the
reference checkout's src/, assembled like the reference's JS assembles it, run on oracle/ref/glsl_rt.h).

    RFX_REFERENCE_DIR=<reference checkout> python tests/golden/make_golden.py [chains] [pins]    # default: both

The reference ships no golden vectors of its own (SURVEY.md §4/§8c); these are outputs of the reference itself run here.
tests/test_oracle_chain_cpu.py checks the C++ oracle against them on any machine (no checkout needed), the `-m gpu` tests check
the CUDA engine against them.  Inputs are stored with the outputs so the fixtures do not depend on the synthetic generator.
  chain_96x54.npz      SSGI chain (K1 -> K2 -> K3 x2 -> K4), 2 frames, steps 12 / refine 3  + K5..K9 and the AO denoise on frame 1
  chain_ssr_64x36.npz  SSR chain (mode "ssr": 1-plane K2/K3, TYPE_SPECULAR compose), 3 frames
  reference_pins.json  every reference-shader call of the pinning tests (tests/test_reference_glsl.py, tests/test_ingest_cpu.py,
                       tests/test_denoiser_options_cpu.py, tests/test_march_options_cpu.py,
                       tests/test_compose_options_cpu.py, tests/test_post_options_cpu.py), in
                       call order (tests/refpins.py); minting runs those tests against the live shaders, so it also checks them
  reference_js_tables.json  the option tables and the export list of the reference's JS (tests/test_host_logic.py)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import chain_harness as ch  # noqa: E402
import refglsl as ref  # noqa: E402  (the reference shaders; NOT the oracle)
from realism_effects_b200 import abi  # noqa: E402


def store_inputs(d, inp):
    d.update(env_map=inp.env_map, env_marginal=inp.env_marginal, env_conditional=inp.env_conditional, env_total=np.float64(inp.env_total))
    for t, fr in enumerate(inp.frames):
        for k in ("depth", "gbuffer", "velocity", "direct"):
            d[f"f{t}_{k}"] = fr[k]
        for k, v in fr["cam"].items():
            d[f"f{t}_cam_{k}"] = np.asarray(v)
        d[f"f{t}_moved"] = np.int32(fr["moved"])


def mint_chains():
    o = ch.Opts(steps=12, refine_steps=3)
    inp = ch.make_inputs(96, 54, 2)
    out = ch.run_oracle_chain(inp, o, impl=ref)
    d = {}
    store_inputs(d, inp)
    for t in range(2):
        for k in ("ssgi", "tr0", "tr1", "dn0", "dn1", "composed"):
            d[f"f{t}_out_{k}"] = out[t][k]
    f0, f1 = inp.frames
    H, W = f1["depth"].shape
    ao = ref.hbao(ch.hbao_params(f1["cam"], 4242), f1["depth"], inp.blue, np.zeros((H, W, 4), np.float16))
    d["hbao"] = ao
    d["ao_composed"] = ref.ao_compose(ch.ao_compose_params(), f1["depth"], ao, f1["direct"])
    vel = ch.rotation_velocity_field(W, H, f1["depth"])
    d["mb_velocity"] = vel
    d["motion_blur"] = ref.motion_blur(ch.motion_blur_params(W, H), vel, f1["direct"], inp.blue)
    d["traa_compose"] = ref.traa_compose(f1["direct"])
    d["ao_dn_a"], d["ao_dn_b"] = ch.ao_denoise(ref, f1, inp.blue, ao)
    d["traa_h0"], d["traa_h1"] = ch.traa_two_frames(ref, f0, f1)
    d["k5_plain"] = ref.ssgi_compose(f1["depth"], out[1]["composed"], f1["direct"])
    d["k5_fog"] = ref.ssgi_compose(f1["depth"], out[1]["composed"], f1["direct"], ch.fog_params(f1["cam"], False))
    d["k5_fog_exp2"] = ref.ssgi_compose(f1["depth"], out[1]["composed"], f1["direct"], ch.fog_params(f1["cam"], True))
    path = os.path.join(HERE, "chain_96x54.npz")
    np.savez_compressed(path, **d)
    print("wrote", path, os.path.getsize(path), "bytes")

    o = ch.Opts(mode=abi.MODE_SSR)
    inp = ch.make_inputs(64, 36, 3)
    out = ch.run_oracle_chain(inp, o, impl=ref)
    d = {}
    store_inputs(d, inp)
    for t in range(3):
        for k in ("ssgi", "tr0", "dn0", "composed"):
            d[f"f{t}_out_{k}"] = out[t][k]
    path = os.path.join(HERE, "chain_ssr_64x36.npz")
    np.savez_compressed(path, **d)
    print("wrote", path, os.path.getsize(path), "bytes")


def mint_pins():
    import json

    import refpins
    import test_compose_options_cpu
    import test_denoiser_options_cpu
    import test_host_logic
    import test_ingest_cpu
    import test_march_options_cpu
    import test_post_options_cpu
    import test_reference_glsl as t

    refpins.MINT = True
    for mode in (abi.MODE_SSGI, abi.MODE_SSR):
        t.test_oracle_equals_reference_shaders_chain(mode)
        t.test_oracle_equals_reference_shaders_orthographic_camera(mode)
    t.test_oracle_equals_reference_shaders_effect_passes()
    t.test_oracle_equals_reference_shaders_cosmetic_effects_and_taa()
    t.test_random_option_sets_oracle_equals_reference_shaders()
    test_denoiser_options_cpu.test_oracle_equals_reference_shaders_denoiser_option_space()
    test_march_options_cpu.test_oracle_equals_reference_shaders_march_options()
    test_compose_options_cpu.test_oracle_equals_reference_shaders_compose_options()
    test_post_options_cpu.test_oracle_equals_reference_shaders_post_options()
    test_ingest_cpu.test_oracle_ingest_equals_the_reference_packgbuffer_glsl()
    path = refpins.save()
    print("wrote", path, os.path.getsize(path), "bytes")
    tables = test_host_logic.reference_js_tables(ref.assemble.REF)
    with open(test_host_logic.JS_GOLDEN, "w", encoding="utf-8") as f:
        json.dump(tables, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", test_host_logic.JS_GOLDEN)


def main(which):
    assert ref.assemble.available(), "the reference checkout is needed"
    if "chains" in which:
        mint_chains()
    if "pins" in which:
        mint_pins()


if __name__ == "__main__":
    main(sys.argv[1:] or ("chains", "pins"))
