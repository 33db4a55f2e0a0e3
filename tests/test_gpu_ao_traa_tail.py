"""The AO chain's TRAA frame tail (rfx_ao_chain_enable_traa) on the GPU: the frame an AOEffect user runs with TRAA, K6 / K6h -> Poisson -> K7
into a chain-owned plane, then TRAA (K2 in its TRAA form) and K9 into frame->output.  The chain writes the bytes of HBAOEffect /
HorizonAOEffect followed by TRAAEffect.update and compose launched per pass, stays within the oracle, and a row-sharded group with the
tail equals one chain byte for byte; every status the tail adds is checked."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

import ao_harness as ao
import chain_harness as ch
from realism_effects_b200 import abi, effects, engine, parallel
from test_gpu_ao_chain import HORIZON_SMALL, Cam, Composer, OracleAo, Scene, _attach, _diff, _group_scene

pytestmark = pytest.mark.gpu


class VelocityPass:
    """TRAAEffect's velocityDepthNormalPass: only `.texture` (the frame's velocity plane) is read"""

    def __init__(self):
        self.texture = None


def _new_traa_effect(comp, cam, vel, options):
    """TRAAEffect whose TemporalReprojectPass is built and reset before its first frame: the chain's tail starts with keepData 0
    (rfx_ao_chain_enable_traa), where a TemporalReprojectPass created by TRAAEffect.update starts with the uniform's default 1"""
    fx = effects.TRAAEffect(None, cam, vel, options)
    fx.temporalReprojectPass = effects.TemporalReprojectPass(None, cam, vel, comp.outputBuffer, 1, fx.options)
    fx.reset()
    return fx


def _sequence(inp):
    """(frame, what the host does before it): moving frames 0-2, a still camera for frames 3-4 (fullAccumulate), a reset before frame 5,
    enable_traa again before frame 6 (a still frame)"""
    m = inp.frames
    return [(m[0], None), (m[1], None), (m[2], None), (m[2], None), (m[2], None), (m[3], "reset"), (m[3], "enable")]


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "exact"])
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("use_normal", [False, True], ids=["depth-normal", "normal-plane"])
@pytest.mark.parametrize("iterations", [0, 1, 2])
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
def test_ao_chain_with_the_tail_equals_the_effects(built, horizon, iterations, use_normal, scale, fast):
    """Over 7 frames (moving, still with fullAccumulate, a reset, enable_traa again) the AO target, the denoised plane, the K7 plane, the
    TRAA accumulated plane and the K9 output equal the AO effect followed by TRAAEffect.update and TRAAEffect.compose, byte for byte"""
    W, H = 96, 64
    inp = ch.make_inputs(W, H, 4)
    opts = {"blueNoiseStart": 777, "resolutionScale": scale, "useNormalPass": use_normal, "iterations": iterations, **(HORIZON_SMALL if horizon else {})}
    topt = abi.make_traa_tail_options(full_accumulate=True)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast)
        comp = Composer(ctx, W, H)
        seq = _sequence(inp)
        cam, vel = Cam(seq[0][0]["cam"]), VelocityPass()
        normals = [ao.view_normal_plane(W, H, t, fr["cam"]) if use_normal else None for t, (fr, _) in enumerate(seq)]
        sc = Scene(ctx, seq[0][0], normals[0])
        make_fx = lambda: (effects.HorizonAOEffect if horizon else effects.HBAOEffect)(comp, cam, sc, opts)  # noqa: E731
        fx, traa = make_fx(), _new_traa_effect(comp, cam, vel, {"fullAccumulate": True})
        chain = engine.AoChain(ctx, engine.ao_chain_options(W, H, opts, horizon=horizon))
        chain.enable_traa(topt)
        final, out = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
        prev = None
        for t, (fr, action) in enumerate(seq):
            if action == "reset":  # back to a new chain: a new AO effect and a new (reset) TRAA effect
                chain.reset()
                fx.dispose()
                traa.dispose()
                fx, traa, prev = make_fx(), _new_traa_effect(comp, cam, vel, {"fullAccumulate": True}), None
            if action == "enable":  # new options, same camera history: TemporalReprojectPass.reset()
                chain.enable_traa(topt)
                traa.reset()
            moved = effects._did_camera_move(fr["cam"], prev)
            sc.free()
            sc2 = Scene(ctx, fr, normals[t])
            sc.depth, sc.velocity, sc.normal = sc2.depth, sc2.velocity, sc2.normal
            fx._normal = sc.normal if use_normal else None
            cam.u, vel.texture = fr["cam"], sc.velocity
            comp.inputBuffer.upload(fr["direct"])
            fx.update(None, comp.inputBuffer)            # the AO EffectPass: K7 into the composer's output buffer
            traa.update(None, comp.outputBuffer)         # the TRAA EffectPass
            traa.compose(final)
            chain.render(fr["cam"], sc.depth, sc.velocity, sc.normal, comp.inputBuffer, out, traa_cam=fr["cam"], camera_moved=moved)
            prev = fr["cam"]
            _diff(f"frame {t} AO target", fx.aoTarget.download(), chain.download(0))
            _diff(f"frame {t} denoised", fx.texture.download(), chain.download(1))
            _diff(f"frame {t} K7 plane", comp.outputBuffer.download(), chain.download(2))
            _diff(f"frame {t} TRAA accumulated", traa.temporalReprojectPass.accumulated.download(), chain.download(3))
            got = out.download()
            _diff(f"frame {t} K9 output", final.download(), got)
            assert np.isfinite(got).all() and (got[..., 3] == 1).all()
        chain.close()
        fx.dispose()
        traa.dispose()
    finally:
        ctx.close()


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "exact"])
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
def test_tail_follows_the_oracle(built, horizon, fast):
    """The tail over 3 moving frames vs the oracle's AO chain -> orc.temporal_reproject(out_half=True) -> orc.traa_compose: within the bar of
    test_gpu_traa_tail.py::test_tail_follows_the_oracle (<= 2e-3 of the pixels outside 1e-3); with fast_math off every kernel of the chain and
    of the tail is bit-equal to the oracle, so the K7 plane, the TRAA accumulated plane and the K9 output must equal it byte for byte."""
    import orc

    W, H = 96, 64
    inp = ch.make_inputs(W, H, 3)
    opts = {"blueNoiseStart": 777, "iterations": 1, **(HORIZON_SMALL if horizon else {})}
    topt = abi.make_traa_tail_options()
    oracle = OracleAo(W, H, opts, horizon)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast)
        chain = engine.AoChain(ctx, engine.ao_chain_options(W, H, opts, horizon=horizon))
        chain.enable_traa(topt)
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        hist, keep, prev = np.zeros((H, W, 4), np.float16), 0.0, None
        for t, fr in enumerate(inp.frames):
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            chain.render(fr["cam"], d, v, None, i, out, traa_cam=fr["cam"], camera_moved=fr["moved"])
            k7 = oracle.frame(fr, inp.blue, None, fr["direct"].astype(np.float16))[2]
            tp = ch.traa_temporal_params(abi.make_camera(fr["cam"]), fr["cam"]["position"], prev or fr["cam"], keep)
            hist, _ = orc.temporal_reproject(tp, k7, fr["velocity"], hist, None, hist, None, out_half=True)
            keep, prev = 1.0, fr["cam"]
            want = {"K7 plane": (k7, chain.download(2)), "TRAA accumulated": (hist, chain.download(3)), "K9 output": (orc.traa_compose(hist), out.download())}
            for name, (w, g) in want.items():
                if not fast:
                    assert not ch.byte_report("", w, g), ch.byte_report(f"frame {t} {name}", w, g)
                c = ch.compare(w, g)
                assert c["frac_bad"] <= 2e-3, (t, name, c)
            for p in (d, v, i):
                p.free()
        chain.close()
    finally:
        ctx.close()


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "exact"])
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
@pytest.mark.parametrize("world", [2, 3, 4, 5, 8])
def test_inprocess_group_with_the_tail_is_bit_identical_to_one_chain(built, world, horizon, fast):
    """N bands on one GPU with the tail (K7 widened by RFX_TRAA_TAIL_ROWS, the TRAA history read on the member that owns the row; with
    fast_math off the exact peer form of the TRAA pass): the wide-FOV scene whose sky silhouette crosses the borders, borders moved down at
    frame 2 and up at frame 4, a still frame at the end (fullAccumulate).  Outputs 0..3 and the K9 frame equal one chain's on every frame."""
    W, H, inp, bg = _group_scene(world, 5)
    frames = inp.frames[:4] + [inp.frames[3]]
    opts = {"iterations": 2, "useNormalPass": world % 2 == 1, **(HORIZON_SMALL if horizon else {})}
    topt = abi.make_traa_tail_options(full_accumulate=True)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast)
        copt = engine.ao_chain_options(W, H, opts, horizon=horizon)
        single = engine.AoChain(ctx, copt)
        single.enable_traa(topt)
        grp = parallel.InProcessAoGroup(ctx, copt, world, traa=topt)
        b = list(grp.bounds)
        if world >= 3:
            assert any(0.0 < bg[max(0, x - 20):x + 20].mean() < 1.0 for x in b[1:-1])
        out1, outg = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
        prev = None
        for t, fr in enumerate(frames):
            if t == 2:
                grp.set_bounds([0] + [x + 16 for x in b[1:-1]] + [H])
            if t == 4:
                grp.set_bounds([0] + [x - 16 for x in b[1:-1]] + [H])
            moved = effects._did_camera_move(fr["cam"], prev)
            prev = fr["cam"]
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            n = ctx.upload(ao.view_normal_plane(W, H, t, fr["cam"])) if opts["useNormalPass"] else None
            single.render(fr["cam"], d, v, n, i, out1, traa_cam=fr["cam"], camera_moved=moved)
            grp.render(fr["cam"], d, v, n, i, outg, traa_cam=fr["cam"], camera_moved=moved)
            for which in (0, 1, 2, 3):
                _diff(f"world {world} frame {t} output {which} bounds {grp._last_bounds}", single.download(which), grp.download(which))
            _diff(f"world {world} frame {t} K9 output", out1.download(), outg.download())
            for p in (d, v, i, n):
                if p is not None:
                    p.free()
        grp.close()
        single.close()
    finally:
        ctx.close()


def test_statuses(built):
    W, H = 128, 256
    inp = ch.make_inputs(W, H, 2)
    fr = inp.frames[0]
    ctx = engine.Context(0, inp.blue)
    lib = ctx.lib
    try:
        copt = engine.ao_chain_options(W, H, {"iterations": 1})
        d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        chain = engine.AoChain(ctx, copt)
        f = chain._frame(fr["cam"], d, v, None, i, out)
        tf = chain._traa_frame(fr["cam"], True)
        # the AO tail has no K5: `compose` must be all zero
        bad = abi.make_traa_tail_options(compose=ch.fog_params(fr["cam"], exp2=False))
        assert lib.rfx_ao_chain_enable_traa(chain.h, C.byref(bad)) == 1
        # tail off: the new entry points are not ready, outputs 2 / 3 stay invalid
        assert lib.rfx_ao_chain_render_traa(chain.h, None, C.byref(f), C.byref(tf)) == 5
        for which in (2, 3):
            assert lib.rfx_ao_chain_output(chain.h, which, C.byref(abi.Plane())) == 1
        chain.render(fr["cam"], d, v, None, i, out)
        # tail on: the old entry point lacks the camera; input and output are required; no TRAA frame is an argument error
        chain.enable_traa()
        assert lib.rfx_ao_chain_render(chain.h, None, C.byref(f)) == 1
        assert lib.rfx_ao_chain_render_traa(chain.h, None, C.byref(chain._frame(fr["cam"], d, v, None, i, None)), C.byref(tf)) == 1
        assert lib.rfx_ao_chain_render_traa(chain.h, None, C.byref(chain._frame(fr["cam"], d, v, None, None, out)), C.byref(tf)) == 1
        assert lib.rfx_ao_chain_render_traa(chain.h, None, C.byref(f), None) == 1
        assert lib.rfx_ao_chain_render_traa(chain.h, None, C.byref(f), C.byref(tf)) == 0
        assert chain.download(2).shape == chain.download(3).shape == (H, W, 4)
        # set_options does not reset the TRAA history: with the call between two frames a chain renders the bytes of one without it
        twins = [engine.AoChain(ctx, copt) for _ in range(2)]
        twin_out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        for c, o in zip(twins, (out, twin_out)):
            c.enable_traa()
            c.render(fr["cam"], d, v, None, i, o, traa_cam=fr["cam"])
        twins[0].set_options(copt)
        f1 = inp.frames[1]
        for c, o in zip(twins, (out, twin_out)):
            c.render(f1["cam"], d, v, None, i, o, traa_cam=f1["cam"])
        _diff("set_options keeps the TRAA history", twins[1].download(3), twins[0].download(3))
        _diff("set_options keeps the TRAA history (K9)", twin_out.download(), out.download())
        for c in twins:
            c.close()
        # NULL turns the tail off: outputs 2 / 3 invalid again, the old entry point renders
        chain.enable_traa(enable=False)
        assert lib.rfx_ao_chain_output(chain.h, 2, C.byref(abi.Plane())) == 1
        assert lib.rfx_ao_chain_render(chain.h, None, C.byref(f)) == 0
        chain.close()
        # groups: members that disagree on the tail; a member of a group of n > 1 cannot change its tail; the sharded entry points
        a, b = engine.AoChain(ctx, copt), engine.AoChain(ctx, copt)
        a.enable_traa()
        st, groups = _attach(ctx, [a, b])
        assert st == 1 and "TRAA tail" in lib.rfx_last_error(ctx.h).decode()
        for g in groups:
            lib.rfx_group_destroy(g)
        a.close()
        b.close()
        grp = parallel.InProcessAoGroup(ctx, copt, 2)
        m = grp.chains[0]
        assert lib.rfx_ao_chain_enable_traa(m.h, C.byref(abi.make_traa_tail_options())) == abi.ERR_UNSUPPORTED
        assert lib.rfx_ao_chain_render_sharded_traa(m.h, None, C.byref(m._frame(fr["cam"], d, v, None, i, out)), C.byref(tf)) == 5
        grp.close()
        grp = parallel.InProcessAoGroup(ctx, copt, 2, traa=abi.make_traa_tail_options())
        m = grp.chains[0]
        assert lib.rfx_ao_chain_render_sharded(m.h, None, C.byref(m._frame(fr["cam"], d, v, None, i, out))) == 1
        grp.close()
        for p in (d, v, i, out, twin_out):
            p.free()
    finally:
        ctx.close()


# ---- two processes, one GPU each (CUDA-IPC peer mappings or the NCCL all-gather fallback) ------------------------------------------------
def _worker(rank, world, port, q, case):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    if case.get("exchange"):
        os.environ["RFX_GROUP_EXCHANGE"] = case["exchange"]
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        inp = ch.make_inputs(case["w"], case["h"], case["frames"], fov=75.0)
        ctx = engine.Context(rank, inp.blue)
        ctx.set_fast_math(case["fast"])
        sh = parallel.ShardedAoChain(ctx, engine.ao_chain_options(case["w"], case["h"], case["opts"]), rebalance_every=1, rebalance_lag=1,
                                     traa=abi.make_traa_tail_options())
        assert sh.uses_peer_reads == (case.get("exchange") != "allgather")
        rows = []
        for fr in inp.frames:
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            out = ctx.alloc(abi.FMT_RGBA16F, case["w"], case["h"])
            sh.render(fr["cam"], d, v, None, i, out, traa_cam=fr["cam"], camera_moved=fr["moved"])
            b0, b1 = sh.band_of_last_frame
            got = {w: sh.chain.download(w)[b0:b1].tobytes() for w in (0, 1, 2, 3)}
            got["out"] = out.download()[b0:b1].tobytes()
            rows.append(((b0, b1), got))
            for p in (d, v, i, out):
                p.free()
        q.put((rank, rows))
        sh.close()
        ctx.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("fast", [True, False], ids=["fast", "exact"])
@pytest.mark.parametrize("exchange", [None, "allgather"])
def test_two_gpu_group_with_the_tail_equals_one_gpu(built, exchange, fast):
    """Two processes with cost-driven borders that move every frame: each rank's rows of outputs 0..3 and the K9 frame equal one GPU's"""
    import torch.multiprocessing as mp

    case = dict(w=256, h=256, frames=4, exchange=exchange, fast=fast, opts={"iterations": 1})
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    procs = [mpc.Process(target=_worker, args=(r, 2, port, q, case)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=900) for _ in procs)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    inp = ch.make_inputs(case["w"], case["h"], case["frames"], fov=75.0)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast)
        single = engine.AoChain(ctx, engine.ao_chain_options(case["w"], case["h"], case["opts"]))
        single.enable_traa()
        out = ctx.alloc(abi.FMT_RGBA16F, case["w"], case["h"])
        for t, fr in enumerate(inp.frames):
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            single.render(fr["cam"], d, v, None, i, out, traa_cam=fr["cam"], camera_moved=fr["moved"])
            want = {w: single.download(w) for w in (0, 1, 2, 3)}
            want["out"] = out.download()
            for rank in range(2):
                (b0, b1), got = res[rank][t]
                for w, data in got.items():
                    assert data == want[w][b0:b1].tobytes(), (exchange, t, rank, w)
            for p in (d, v, i):
                p.free()
        single.close()
    finally:
        ctx.close()
