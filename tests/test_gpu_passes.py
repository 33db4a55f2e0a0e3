"""GPU parity tests, pass by pass, through the C ABI.  Each kernel is fed the ORACLE's intermediate planes so errors do
not compound, and is compared with the oracle's output of the same pass.  Plus: golden fixtures (no oracle at run time),
row-block sharding invariance, full-size (4K) properties and the ABI's error behaviour."""
import numpy as np
import pytest

import chain_harness as ch
from realism_effects_b200 import abi, engine, synth

pytestmark = pytest.mark.gpu

MAX_BAD = 1e-4  # fraction of pixels allowed outside 1e-3 relative per pass (1e-4 = 2 pixels of these planes)


def check(name, want, got, packed=False, max_bad=MAX_BAD):
    c = ch.compare(want, got, packed=packed)
    print(f"{name}: bad={c['frac_bad']:.2e} max_rel_ok={c['max_rel_ok']:.1e} bit_equal={c['bit_equal']:.4f}")
    assert c["frac_bad"] <= max_bad, (name, c)
    return c


@pytest.fixture(scope="module")
def scene(built):
    o = ch.Opts(denoise_iterations=2)
    inp = ch.make_inputs(200, 120, 3)
    ref = ch.run_oracle_chain(inp, o)
    return o, inp, ref


@pytest.fixture()
def ctx(built, scene):
    o, inp, _ = scene
    c = engine.Context(0, inp.blue)
    c.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    yield c
    c.close()


def test_k1_ssgi_trace_isolated(scene, ctx):
    o, inp, ref = scene
    for t in (0, 2):
        fr, rec = inp.frames[t], ref[t]
        out = ctx.alloc(abi.FMT_RGBA32F, inp.width, inp.height)
        ctx.ssgi_trace(rec["_k1_params"], ctx.upload(fr["depth"]), ctx.upload(fr["gbuffer"]), None, ctx.upload(fr["direct"]),
                       ctx.upload(rec["_k1_accumulated"]), out)
        check(f"K1 f{t}", rec["ssgi"], out.download(), packed=True)


def test_k1_with_velocity_plane_and_ssr_mode(scene, ctx):
    """non-NULL velocity sampler (intended wiring, SURVEY.md D4) and mode = SSR."""
    import orc

    o, inp, ref = scene
    fr, rec = inp.frames[2], ref[2]
    env = orc.Env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    for mode in (abi.MODE_SSGI, abi.MODE_SSR):
        p = ch.ssgi_params(ch.Opts(mode=mode), abi.make_camera(fr["cam"]), 991, (inp.env_map.shape[1], inp.env_map.shape[0]))
        want = orc.ssgi_trace(p, fr["depth"], fr["gbuffer"], fr["velocity"], fr["direct"], rec["_k1_accumulated"], env, inp.blue)
        out = ctx.alloc(abi.FMT_RGBA32F, inp.width, inp.height)
        ctx.ssgi_trace(p, ctx.upload(fr["depth"]), ctx.upload(fr["gbuffer"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"]),
                       ctx.upload(rec["_k1_accumulated"]), out)
        got = out.download()
        if mode == abi.MODE_SSGI:
            check("K1 velocity", want, got, packed=True)
        else:
            check("K1 ssr rgb", want[..., :3], got[..., :3])
            assert (want[..., 3].view(np.uint32) != got[..., 3].view(np.uint32)).mean() <= MAX_BAD  # packed (rayLength, roughness) halves


def test_k2_temporal_isolated(scene, ctx):
    o, inp, ref = scene
    for t in (0, 1, 2):
        fr, rec = inp.frames[t], ref[t]
        o0, o1 = ctx.upload(rec["_k2_prev_out"][0]), ctx.upload(rec["_k2_prev_out"][1])
        ctx.temporal_reproject(rec["_k2_params"], ctx.upload(rec["ssgi"]), ctx.upload(fr["velocity"]), ctx.upload(rec["_k2_hist"][0]),
                               ctx.upload(rec["_k2_hist"][1]), o0, o1)
        check(f"K2 f{t} diffuse", rec["tr0"], o0.download())
        check(f"K2 f{t} specular", rec["tr1"], o1.download())


def test_k3_poisson_isolated(scene, ctx):
    o, inp, ref = scene
    fr, rec = inp.frames[2], ref[2]
    d, g = ctx.upload(fr["depth"]), ctx.upload(fr["gbuffer"])
    for i, k3 in enumerate(rec["_k3"]):
        o0, o1 = ctx.upload(k3["prev0"]), ctx.upload(k3["prev1"])
        ctx.poisson_denoise(k3["params"], d, g, ctx.upload(k3["in0"]), ctx.upload(k3["in1"]), o0, o1)
        check(f"K3 pass {i} diffuse", k3["out0"], o0.download())
        check(f"K3 pass {i} specular", k3["out1"], o1.download())


def test_k4_compose_isolated(scene, ctx):
    o, inp, ref = scene
    fr, rec = inp.frames[1], ref[1]
    out = ctx.upload(rec["_k4_prev"])
    ctx.gi_compose(rec["_k4_params"], ctx.upload(fr["depth"]), ctx.upload(fr["gbuffer"]), ctx.upload(rec["dn0"]), ctx.upload(rec["dn1"]), out)
    check("K4", rec["composed"], out.download())


def test_k3_single_plane_velocity_layout(scene, ctx):
    """AO denoise configuration: 1 plane, normals/depth from a velocity-layout plane (no GBUFFER_TEXTURE), SURVEY.md D3/P1."""
    import orc

    o, inp, ref = scene
    fr, rec = inp.frames[1], ref[1]
    p = ch.poisson_params(ch.Opts(), 555, True)
    p.texture_count, p.gbuffer_texture, p.input_linear = 1, 0, 1
    p.is_texture_specular[:] = [0, 0]
    p.normal_phi, p.depth_phi = 3.25, 2.0  # PoissonDenoisePass defaults :16-24
    z = np.zeros((inp.height, inp.width, 4), np.float16)
    want, _ = orc.poisson_denoise(p, fr["depth"], fr["velocity"], rec["dn0"], None, inp.blue, z, None)
    out = ctx.upload(z)
    ctx.poisson_denoise(p, ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(rec["dn0"]), None, out, None)
    check("K3 1-plane", want, out.download())


def test_traa_temporal_one_plane(scene, ctx):
    """K2 in its TRAA configuration: 1 RGBA16F plane, inputType DIFFUSE, no background discard (A7)."""
    import orc

    o, inp, ref = scene
    f0, f1 = inp.frames[1], inp.frames[2]
    cam = abi.make_camera(f1["cam"])
    p = ch.traa_temporal_params(cam, f1["cam"]["position"], f0["cam"], 1.0)
    hist = f0["direct"]
    z = np.zeros((inp.height, inp.width, 4), np.float16)
    want, _ = orc.temporal_reproject(p, f1["direct"], f1["velocity"], hist, None, z, None, out_half=True)
    out = ctx.upload(z)
    ctx.temporal_reproject(p, ctx.upload(f1["direct"]), ctx.upload(f1["velocity"]), ctx.upload(hist), None, out, None)
    got = out.download()
    check("K2 TRAA", want, got)
    assert (got[..., 3] > 0).mean() > 0.5
    want9 = orc.traa_compose(want)
    o9 = ctx.alloc(abi.FMT_RGBA16F, inp.width, inp.height)
    ctx.traa_compose(ctx.upload(want), o9)
    assert np.array_equal(want9.view(np.uint16), o9.download().view(np.uint16))


def test_hbao_ao_compose_motion_blur(scene, ctx):
    import orc

    o, inp, ref = scene
    fr = inp.frames[1]
    H, W = inp.height, inp.width
    z = np.zeros((H, W, 4), np.float16)
    hp = ch.hbao_params(fr["cam"], 4242)
    want = orc.hbao(hp, fr["depth"], inp.blue, z)
    out = ctx.upload(z)
    ctx.hbao(hp, ctx.upload(fr["depth"]), out)
    assert out.download().view(np.uint16).tobytes() == want.view(np.uint16).tobytes(), "K6 hbao differs from the oracle"
    ap = ch.ao_compose_params()
    oc = ctx.alloc(abi.FMT_RGBA16F, W, H)
    ctx.ao_compose(ap, ctx.upload(fr["depth"]), ctx.upload(want), ctx.upload(fr["direct"]), oc)
    want7 = orc.ao_compose(ap, fr["depth"], want, fr["direct"])
    assert oc.download().view(np.uint16).tobytes() == want7.view(np.uint16).tobytes(), "K7 ao_compose differs from the oracle"


@pytest.mark.parametrize("frame_index,res", [(7, None), (0, None), (7, (333, 200))])
def test_motion_blur_c1(built, frame_index, res):
    """BASELINE config C1: MotionBlurEffect 256x256, rigid-rotation velocity field; frame 0 = tiled blue-noise lookup;
    `resolution` = window size different from the buffer size (A10)."""
    import orc

    W = H = 256
    fr = synth.render_frame(W, H, 1)
    depth, color = fr.depth.numpy(), fr.direct_light.numpy()
    vel = ch.rotation_velocity_field(W, H, depth)
    blue = synth.load_blue_noise()
    p = ch.motion_blur_params(W, H, frame=frame_index, resolution=res)
    want = orc.motion_blur(p, vel, color, blue)
    c = engine.Context(0, blue)
    try:
        out = c.alloc(abi.FMT_RGBA16F, W, H)
        c.motion_blur(p, c.upload(vel), c.upload(color), out)
        got = out.download()
    finally:
        c.close()
    check("K8 motion blur", want, got)
    assert np.array_equal(got[:8, :8].view(np.uint16), color[:8, :8].view(np.uint16))  # did-not-move early out returns inputColor


def test_chain_matches_golden_fixture(built):
    """CUDA chain vs the committed golden outputs — OUTPUTS OF THE REFERENCE'S OWN SHADERS run on the CPU (tests/golden/make_golden.py ->
    tests/refglsl.py) — no oracle here."""
    from test_oracle_chain_cpu import load_golden

    g, inp = load_golden()
    got, launches = ch.run_cuda_chain(inp, ch.Opts(steps=12, refine_steps=3))
    assert launches >= 2 * (1 + 1 + 2 + 1)  # + env mip chain + per-frame G-buffer decode
    for t in range(2):
        for k in ("ssgi", "tr0", "tr1", "dn0", "dn1", "composed"):
            check(f"golden f{t}.{k}", g[f"f{t}_out_{k}"], got[t][k], packed=(k == "ssgi"), max_bad=6e-3)  # chain-level bar at this small size (one differently resolved ray = ~1e-2 of 5 184 pixels would fail it: none measured)


def test_ssr_chain_and_exact_k1_match_reference_shader_goldens(built):
    """mode "ssr" over 3 frames against the reference shaders' outputs (tests/golden/chain_ssr_64x36.npz), both variants; and in SSGI mode
    (where K1's output is quantised to fp16 pairs) the exact variant's K1 plane is BIT-equal to what the reference's ssgi.frag produced.
    (In SSR mode K1 writes full fp32 colours; the exact variant is within an ulp or two of the reference there.)"""
    from test_oracle_chain_cpu import GOLD_SSR, load_golden

    g, inp = load_golden(GOLD_SSR, 3, (64, 36))
    for fast in (True, False):
        got, _ = ch.run_cuda_chain(inp, ch.Opts(mode=abi.MODE_SSR), capture=("ssgi", "tr0", "dn0", "composed"), fast_math=fast)
        for t in range(3):
            check(f"ssr golden fast={fast} f{t}.ssgi", g[f"f{t}_out_ssgi"][..., :3], got[t]["ssgi"][..., :3], max_bad=6e-3)
            for k in ("tr0", "dn0", "composed"):
                check(f"ssr golden fast={fast} f{t}.{k}", g[f"f{t}_out_{k}"], got[t][k], max_bad=6e-3)
    g2, inp2 = load_golden()
    got, _ = ch.run_cuda_chain(inp2, ch.Opts(steps=12, refine_steps=3), capture=("ssgi",), fast_math=False)
    assert got[0]["ssgi"].tobytes() == g2["f0_out_ssgi"].tobytes()  # K1 (exact variant) == the reference's ssgi.frag, bit for bit


def test_row_block_sharding_is_exact(scene, ctx):
    """Launching a pass on row blocks [0,r) and [r,H) writes exactly what one full launch writes (SURVEY.md §8e)."""
    o, inp, ref = scene
    fr, rec = inp.frames[2], ref[2]
    H, W = inp.height, inp.width
    d, g, v, dl, acc = (ctx.upload(fr["depth"]), ctx.upload(fr["gbuffer"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"]),
                        ctx.upload(rec["_k1_accumulated"]))
    for split in (37, 64):
        full, parts = ctx.alloc(abi.FMT_RGBA32F, W, H), ctx.alloc(abi.FMT_RGBA32F, W, H)
        ctx.ssgi_trace(rec["_k1_params"], d, g, None, dl, acc, full)
        ctx.ssgi_trace(rec["_k1_params"], d, g, None, dl, acc, parts, rows=(0, split))
        ctx.ssgi_trace(rec["_k1_params"], d, g, None, dl, acc, parts, rows=(split, H))
        assert full.download().tobytes() == parts.download().tobytes()
        k3 = rec["_k3"][1]
        f0, f1, p0, p1 = (ctx.upload(k3["prev0"]), ctx.upload(k3["prev1"]), ctx.upload(k3["prev0"]), ctx.upload(k3["prev1"]))
        i0, i1 = ctx.upload(k3["in0"]), ctx.upload(k3["in1"])
        ctx.poisson_denoise(k3["params"], d, g, i0, i1, f0, f1)
        ctx.poisson_denoise(k3["params"], d, g, i0, i1, p0, p1, rows=(0, split))
        ctx.poisson_denoise(k3["params"], d, g, i0, i1, p0, p1, rows=(split, H))
        assert f0.download().tobytes() == p0.download().tobytes() and f1.download().tobytes() == p1.download().tobytes()
        t0, t1, q0, q1 = (ctx.upload(rec["_k2_prev_out"][0]), ctx.upload(rec["_k2_prev_out"][1]), ctx.upload(rec["_k2_prev_out"][0]),
                          ctx.upload(rec["_k2_prev_out"][1]))
        args = (rec["_k2_params"], ctx.upload(rec["ssgi"]), v, ctx.upload(rec["_k2_hist"][0]), ctx.upload(rec["_k2_hist"][1]))
        ctx.temporal_reproject(*args, t0, t1)
        ctx.temporal_reproject(*args, q0, q1, rows=(0, split))
        ctx.temporal_reproject(*args, q0, q1, rows=(split, H))
        assert t0.download().tobytes() == q0.download().tobytes() and t1.download().tobytes() == q1.download().tobytes()


def test_full_size_4k_properties(built):
    """BASELINE config C3 size: determinism, background/sentinel rules and finite outputs at 3840x2160 (oracle-free)."""
    import torch

    W, H = 3840, 2160
    o = ch.Opts(denoise_iterations=2)
    env = synth.synthetic_env(256, 128)
    marg, cond, total = synth.build_env_cdf(env.astype(np.float32))
    frames = [synth.render_frame(W, H, t, device="cuda") for t in (1, 2)]
    outs = []
    for rep in range(2):
        c = engine.Context(0)
        c.set_env(env, marg, cond, total)

        class I:
            width, height = W, H

        chain = engine.SsgiChain(c, ch.chain_options(I, o))
        for fr in frames:
            pl = [c.upload(x.cpu().numpy()) for x in (fr.depth, fr.gbuffer, fr.velocity, fr.direct_light)]
            chain.render(abi.make_camera(fr.cam.uniforms()), *pl, fr.cam.uniforms()["position"], True)
            c.sync()
            for p in pl:
                p.free()
        outs.append({k: chain.download(w) for k, w in (("composed", 0), ("ssgi", 1), ("dn0", 4))})
        chain.close()
        c.close()
    for k in outs[0]:
        assert outs[0][k].tobytes() == outs[1][k].tobytes(), k  # bit-deterministic
    comp, ssgi = outs[0]["composed"], ch.unpack_halves(outs[0]["ssgi"])
    depth = frames[1].depth.cpu().numpy()
    bg = depth == 1.0
    fg_written = comp[~bg][:, 3] == 1.0
    assert fg_written.all(), "every non-discarded pixel is written with alpha 1"
    assert np.isfinite(comp[~bg]).all()
    assert (comp[~bg][:, :3] >= -1e-6).all()  # exp(x)-1 of a ~0 log-average may round a hair below 0
    def interior(b):
        return b & np.roll(b, 1, 0) & np.roll(b, -1, 0) & np.roll(b, 1, 1) & np.roll(b, -1, 1)

    bg_prev = frames[0].depth.cpu().numpy() == 1.0
    never_written = interior(bg) & interior(bg_prev)            # discarded in both frames => the zero-initialised target is untouched;
    assert (comp[never_written] == 0).all()                     # pixels that were foreground last frame keep their stale texel (SURVEY.md A2)
    assert never_written.any()
    assert np.allclose(ssgi[bg][:, :4], ssgi[bg][:, 4:], atol=0)  # background = packTwoVec4(directLight, directLight)
    torch.cuda.synchronize()


def test_abi_error_behaviour(built):
    c = engine.Context(0)
    try:
        d = c.alloc(abi.FMT_R32F, 64, 32)
        g = c.alloc(abi.FMT_RGBA32F, 64, 32)
        out = c.alloc(abi.FMT_RGBA32F, 64, 32)
        p = ch.ssgi_params(ch.Opts(), abi.make_camera(synth.Camera().uniforms()), 5, (64, 32))
        with pytest.raises(abi.RfxError, match="env map"):      # env requested but never set
            c.ssgi_trace(p, d, g, None, None, None, out)
        with pytest.raises(abi.RfxError, match="RGBA32F"):      # wrong format
            c.ssgi_trace(p, d, d, None, None, None, out)
        small = c.alloc(abi.FMT_RGBA32F, 32, 32)
        p.flags = 0
        with pytest.raises(abi.RfxError, match="must have one size"):   # the INPUT planes share one size ...
            c.ssgi_trace(p, d, small, None, None, None, out)
        big = c.alloc(abi.FMT_RGBA32F, 128, 64)
        with pytest.raises(abi.RfxError, match="not larger"):           # ... and the target may be smaller (resolutionScale < 1), never larger
            c.ssgi_trace(p, d, g, None, None, None, big)
        pp = ch.poisson_params(ch.Opts(), 3, True)
        h = c.alloc(abi.FMT_RGBA16F, 64, 32)
        with pytest.raises(abi.RfxError, match="in-place"):
            c.poisson_denoise(pp, d, g, h, h, h, h)
        assert c.launch_count == 0
        c.ssgi_trace(p, d, g, None, None, None, out)             # flags = 0: no env needed
        c.sync()
        assert c.launch_count == 2                               # viewZ prepass + trace
    finally:
        c.close()
