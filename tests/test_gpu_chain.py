"""GPU parity of the whole SSGI chain (K1 -> K2 -> K3 x n -> K4) through the C ABI vs the oracle, for both kernel
variants: fast_math=True (SFU lg2/ex2; the default, what bench.py times) and fast_math=False (correctly rounded transcendentals, every
plane byte-equal to the oracle)."""
import numpy as np
import pytest

import chain_harness as ch
from realism_effects_b200 import abi

pytestmark = pytest.mark.gpu

CASES = [
    dict(width=192, height=108, frames=3),
    dict(width=161, height=91, frames=2, denoise_iterations=2),            # odd sizes: helper lanes beyond the edge
    dict(width=128, height=72, frames=2, importance_sampling=False),
    dict(width=128, height=72, frames=2, use_envmap=False, use_direct_light=False, steps=8, refine_steps=0),
    dict(width=128, height=72, frames=2, missed_rays=True),
    dict(width=160, height=90, frames=3, mode=1),                         # SSR: 1 plane, K4 with inputType "specular" (scene colour + specular GI * F)
    dict(width=128, height=72, frames=2, mode=1, denoise_iterations=0),   # SSR without Poisson passes
]


@pytest.mark.parametrize("fast", [True, False])
@pytest.mark.parametrize("kw", CASES)
def test_chain_parity(built, kw, fast):
    res = ch.run_chain_parity(fast_math=fast, **kw)
    print(res["summary"])
    assert res["ok"], res["summary"]
    assert res["launches"] > 0


def test_ssr_chain_writes_composed_and_feeds_it_back(built):
    """SSR mode end to end (ADVICE r1): `composed` = sceneTexture + specularGi * F + emissive is written every frame and is what
    the next frame's hit rays sample (src/ssgi/pass/SSGIPass.js:88) — it must not stay zero."""
    o = ch.Opts(mode=1)
    inp = ch.make_inputs(160, 90, 3)
    ref = ch.run_oracle_chain(inp, o)
    got, _ = ch.run_cuda_chain(inp, o)
    for t in range(3):
        assert np.abs(got[t]["composed"][..., :3]).max() > 0.05
        c = ch.compare(ref[t]["composed"], got[t]["composed"])
        assert c["frac_bad"] <= 6e-3, (t, c)
    assert not np.array_equal(got[1]["ssgi"], got[0]["ssgi"])


def test_static_camera_full_accumulate(built):
    """static camera => fullAccumulate path (TemporalReprojectPass.js:178-180), history length grows every frame"""
    o = ch.Opts()
    inp = ch.make_inputs(160, 90, 4, static=True)
    ref = ch.run_oracle_chain(inp, o)
    got, _ = ch.run_cuda_chain(inp, o)
    for t in range(4):
        for k in ("tr0", "tr1", "composed"):
            c = ch.compare(ref[t][k], got[t][k])
            assert c["frac_bad"] <= 6e-3 and ch.compare(ref[t][k], got[t][k], rtol=4e-3)["frac_bad"] <= 1.5e-3, (t, k, c)  # chain-level bar, see chain_harness
    assert got[3]["tr0"][..., 3].max() > got[1]["tr0"][..., 3].max()


def test_host_buffer_paths_match_device_path(built):
    """rfx_ssgi_chain_render_host and the pipelined submit_host / wait_host pair give, frame for frame, the bytes of the
    device-plane path (same kernels, only the copies and the stream/event ordering differ)."""
    import ctypes as C

    from realism_effects_b200 import abi, engine

    o = ch.Opts(denoise_iterations=1)
    inp = ch.make_inputs(160, 96, 5)
    want, _ = ch.run_cuda_chain(inp, o, capture=("composed",))
    for pipelined in (False, True):
        ctx = engine.Context(0, inp.blue)
        try:
            ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
            chain = engine.SsgiChain(ctx, ch.chain_options(inp, o))
            outs = [np.zeros((inp.height, inp.width, 4), np.float32) for _ in inp.frames]
            keep = []
            for i, fr in enumerate(inp.frames):
                hf = abi.SsgiHostFrame()
                hf.cam = abi.make_camera(fr["cam"])
                bufs = [np.ascontiguousarray(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
                keep.append(bufs)  # pageable host memory is fine (slower, still ordered); buffers stay alive until the frame completed
                hf.depth, hf.gbuffer, hf.velocity, hf.direct_light = (b.ctypes.data_as(C.c_void_p).value for b in bufs)
                hf.camera_pos[:] = [float(x) for x in fr["cam"]["position"]]
                hf.camera_moved = int(fr["moved"])
                hf.out_composed = outs[i].ctypes.data_as(C.c_void_p).value
                if pipelined:
                    chain.submit_host(hf)
                    chain.wait_host(1)
                else:
                    chain.render_host(hf)
            chain.wait_host(0)
            for i in range(len(inp.frames)):
                assert outs[i].tobytes() == want[i]["composed"].tobytes(), f"frame {i} pipelined={pipelined}"
            chain.close()
        finally:
            ctx.close()


def test_group_of_one_rank_equals_plain_chain(built):
    """rfx_group_* with world = 1 on a single GPU: NCCL is loaded and initialised, the chain is attached, every frame ends with the
    group's collective, the band is the whole frame — and the bytes are those of rfx_ssgi_chain_render.  (The peer-mapped reads need
    >= 2 GPUs: tests/test_gpu_multi.py; this keeps the group plumbing covered on a 1-GPU box.)"""
    import ctypes as C

    from realism_effects_b200 import abi, engine, parallel

    o = ch.Opts(denoise_iterations=1)
    inp = ch.make_inputs(160, 128, 3)
    want, _ = ch.run_cuda_chain(inp, o)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        buf = C.create_string_buffer(abi.GROUP_ID_BYTES)
        ctx._chk(ctx.lib.rfx_group_get_unique_id(buf))
        sh = parallel.ShardedSsgiChain(ctx, ch.chain_options(inp, o), rank=0, world=1, unique_id=bytes(buf.raw), rebalance_every=1, rebalance_lag=1)
        assert sh.bounds == (0, 128)
        keep = []
        for t, fr in enumerate(inp.frames):
            pl = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            keep.append(pl)
            sh.render(abi.make_camera(fr["cam"]), *pl, fr["cam"]["position"], fr["moved"])
            for k, which in (("composed", 0), ("ssgi", 1), ("tr0", 2), ("dn1", 5)):
                assert sh.chain.download(which).tobytes() == want[t][k].tobytes(), (t, k)
        assert len(sh.last_costs) == 1
        sh.close()
    finally:
        ctx.close()


def test_tma_staged_poisson_passes_are_bit_identical(built, monkeypatch):
    """The TMA-staged Poisson passes (cpoisson_tma_kernel: tap tiles through cp.async.bulk.tensor + mbarrier into shared memory,
    default on) write exactly the bytes of the global-load path (RFX_K3_TMA=0) — frames large enough to have interior blocks, with
    background regions, over several frames so the history feeds back."""
    o = ch.Opts(denoise_iterations=2)
    inp = ch.make_inputs(320, 192, 3)
    outs = {}
    for tma in ("1", "0"):
        monkeypatch.setenv("RFX_K3_TMA", tma)
        outs[tma], _ = ch.run_cuda_chain(inp, o)
    for t in range(3):
        for k in ("dn0", "dn1", "composed", "tr0"):
            assert outs["1"][t][k].tobytes() == outs["0"][t][k].tobytes(), (t, k)


@pytest.mark.parametrize("mode", [abi.MODE_SSGI, abi.MODE_SSR])
@pytest.mark.parametrize("denoise_mode", [abi.DENOISE_FULL_TEMPORAL, abi.DENOISE_TEMPORAL])
def test_chain_denoise_modes_full_temporal_and_temporal(built, mode, denoise_mode):
    """option denoiseMode (src/denoise/Denoiser.js:7,45-78): "full_temporal" (what preset "low" selects: K2 -> K4 on the temporal textures, the history
    is the RGBA32F FramebufferTexture copy of the temporal target for BOTH planes) and "temporal" (K2 only; K1 samples the temporal texture).  3 frames
    with history against the oracle chain (which equals the reference shaders bit for bit in these modes too: tools/pin_oracle.py)."""
    o = ch.Opts(mode=mode, denoise_mode=denoise_mode)
    inp = ch.make_inputs(160, 90, 3)
    planes = ("ssgi", "tr0", "tr1", "composed") if mode == abi.MODE_SSGI else ("ssgi", "tr0", "composed")
    ref = ch.run_oracle_chain(inp, o, capture=planes, lean=True)
    for fast in (True, False):
        got, launches = ch.run_cuda_chain(inp, o, capture=planes, fast_math=fast)
        for t in range(3):
            for k in planes:
                if not fast:
                    assert not ch.byte_report("", ref[t][k], got[t][k]), ch.byte_report(f"f{t}.{k}", ref[t][k], got[t][k])
                    continue
                a, b = (ref[t][k][..., :3], got[t][k][..., :3]) if (k == "ssgi" and mode == abi.MODE_SSR) else (ref[t][k], got[t][k])
                c = ch.compare(a, b, packed=(k == "ssgi" and mode == abi.MODE_SSGI))
                assert c["frac_bad"] <= 6e-3, (fast, t, k, c)
    with pytest.raises(abi.RfxError):
        bad = ch.chain_options(inp, o)
        bad.denoise_mode = 3  # "denoised": cannot run in the reference either
        from realism_effects_b200 import engine
        ctx = engine.Context(0, inp.blue)
        try:
            engine.SsgiChain(ctx, bad)
        finally:
            ctx.close()


@pytest.mark.parametrize("mode,scale", [(abi.MODE_SSGI, 0.5), (abi.MODE_SSGI, 0.75), (abi.MODE_SSR, 0.5)])
def test_chain_resolution_scale(built, mode, scale):
    """option resolutionScale (src/ssgi/pass/SSGIPass.js:52-57): K1 renders into a (w * scale) x (h * scale) target and samples the full-size G-buffer by
    uv; the temporal pass reads that smaller target NEAREST at full size.  3 frames against the oracle chain (= the reference shaders, bit for bit)."""
    o = ch.Opts(mode=mode, resolution_scale=scale)
    inp = ch.make_inputs(160, 96, 3)
    planes = ("ssgi", "tr0", "tr1", "dn0", "dn1", "composed") if mode == abi.MODE_SSGI else ("ssgi", "tr0", "dn0", "composed")
    ref = ch.run_oracle_chain(inp, o, capture=planes, lean=True)
    assert ref[0]["ssgi"].shape[:2] == (int(96 * scale), int(160 * scale))
    for fast in (True, False):
        got, _ = ch.run_cuda_chain(inp, o, capture=planes, fast_math=fast)
        for t in range(3):
            for k in planes:
                a, b = (ref[t][k][..., :3], got[t][k][..., :3]) if (k == "ssgi" and mode == abi.MODE_SSR) else (ref[t][k], got[t][k])
                assert a.shape == b.shape, (k, a.shape, b.shape)
                if not fast:
                    assert not ch.byte_report("", ref[t][k], got[t][k]), ch.byte_report(f"f{t}.{k}", ref[t][k], got[t][k])
                    continue
                c = ch.compare(a, b, packed=(k == "ssgi" and mode == abi.MODE_SSGI))
                assert c["frac_bad"] <= 8e-3, (fast, t, k, c)


@pytest.mark.parametrize("world", [2, 3, 4, 5, 8])
def test_inprocess_group_of_n_bands_is_bit_identical_to_one_chain(built, world):
    """The row-sharded group's N-band logic on ONE GPU (rfx_group_create_inprocess): every member renders its band with the halo rows recomputed
    locally and reads last frame's history rows on the member that owns them; the assembled frame — every plane — equals the plain chain byte for
    byte over 5 frames, with the band borders moved twice (so rows change owner and carried texels / history come from another member)."""
    from realism_effects_b200 import engine, parallel

    W, H = 320, 64 * world + 112
    o = ch.Opts(denoise_iterations=2)
    inp = ch.make_inputs(W, H, 5, fov=75.0)  # a wide view: the sky's silhouette (discarded pixels next to shaded ones) crosses the band borders
    bg = inp.frames[0]["depth"] == 1.0
    assert 0.15 < bg.mean() < 0.7
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, o)
        single = engine.SsgiChain(ctx, copt)
        grp = parallel.InProcessGroup(ctx, copt, world)
        b = list(grp.bounds)
        assert b[0] == 0 and b[-1] == H and len(b) == world + 1
        if world >= 3:  # at least one interior border runs through the silhouette (rows with both discarded and shaded pixels within the halos)
            assert any(0.0 < bg[max(0, x - 20):x + 20].mean() < 1.0 for x in b[1:-1])
        for t, fr in enumerate(inp.frames):
            if t == 2:  # move every interior border down by 16 rows, then (t == 4) up by 32
                grp.set_bounds([0] + [x + 16 for x in b[1:-1]] + [H])
            if t == 4:
                grp.set_bounds([0] + [x - 16 for x in b[1:-1]] + [H])
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            cam = abi.make_camera(fr["cam"])
            single.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            grp.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            for which, name in ((0, "composed"), (1, "ssgi"), (4, "dn0"), (5, "dn1")):
                a, g = single.download(which), grp.download(which)
                if a.tobytes() != g.tobytes():
                    ne = (a.view(np.uint8).reshape(H, -1) != g.view(np.uint8).reshape(H, -1)).any(1)
                    rows = np.nonzero(ne)[0]
                    raise AssertionError(f"world {world} frame {t} {name}: rows {rows[0]}..{rows[-1]} differ ({len(rows)} rows); bounds {grp._last_bounds}")
            for p in planes:
                p.free()
        grp.close()
        single.close()
    finally:
        ctx.close()
