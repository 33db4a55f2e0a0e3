"""TRAAEffect + MotionBlurEffect as one EffectPass on the GPU: rfx_traa_motion_blur_launch is bit-equal to the oracle over the grid of
tests/test_traa_motion_blur_cpu.py (whose oracle is pinned to the reference's shaders), and the chains' motion-blur stage
(rfx_*_chain_set_motion_blur) writes the bytes of the per-pass effects every frame; every status the stage adds is checked."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

import chain_harness as ch
import mb_harness as mb
from realism_effects_b200 import abi, effects, engine, parallel
from test_gpu_ao_chain import Cam, Composer, Scene, _attach, _diff
from test_gpu_ao_traa_tail import VelocityPass, _new_traa_effect
from test_gpu_post_options import bit_equal, free, one_and_two_launches, uploaded
from test_gpu_traa_tail import _traa_params
from test_post_options_cpu import K8Case
from test_traa_motion_blur_cpu import MB_CASES, mb_call, tap_span

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "exact"])
@pytest.mark.parametrize("case", MB_CASES, ids=str)
def test_traa_motion_blur_matches_the_oracle(built, case: K8Case, fast):
    """one launch and two launches split at an odd row, fast_math on and off (the pass has one form: the same bytes)"""
    p, vel, acc, inp, blue = mb_call(case)
    want = mb.oracle(p, vel, acc, inp, blue)
    ctx = engine.Context(0, blue)
    try:
        ctx.set_fast_math(fast)
        ins = uploaded(ctx, vel, acc, inp)
        try:
            got = one_and_two_launches(ctx, str(case), lambda out, rows: ctx.traa_motion_blur(p, *ins, out, rows=rows), np.zeros_like(inp), inp.shape[0])
        finally:
            free(ins)
        bit_equal(str(case), want, got)
    finally:
        ctx.close()


def _blur_params(t: int, W: int, H: int) -> abi.MotionBlurParams:
    """frame t's MotionBlurEffect uniforms: the frame counter moves on, deltaTime alternates between 1/1000 (long taps) and 1/60"""
    p = ch.motion_blur_params(W, H, frame=t, samples=16, delta_time=1 / 1000 if t % 2 == 0 else 1 / 60)
    p.intensity = 3.0
    return p


@pytest.mark.parametrize("kw", [dict(), dict(mode=abi.MODE_SSR, denoise_mode=1)], ids=["fast-ssgi", "ssr-full_temporal"])
def test_ssgi_chain_with_the_stage_equals_the_per_pass_effects(built, kw):
    """5 moving frames: output 6 == ssgi_compose -> temporal_reproject (TRAA form) -> rfx_traa_motion_blur_launch over the K5 plane,
    launched one by one on the chain's own `composed`, and output 7 == the TRAA accumulated plane, byte for byte"""
    W, H = 160, 96
    inp = ch.make_inputs(W, H, 5)
    ctx = engine.Context(0, inp.blue)
    chain = None
    planes = []
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        chain = engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts(**kw)))
        topt = abi.make_traa_tail_options()
        chain.enable_traa(topt)
        k5, out = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
        acc = [ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)]
        planes = [k5, out] + acc
        keep, prev, blurred = 0.0, None, 0
        for t, fr in enumerate(inp.frames):
            fp = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            p = _blur_params(t, W, H)
            chain.set_motion_blur(p)
            chain.render(abi.make_camera(fr["cam"]), *fp, fr["cam"]["position"], fr["moved"])
            ctx.ssgi_compose(fp[0], chain.output(0), fp[3], k5, params=topt.compose)
            ctx.temporal_reproject(_traa_params(topt, fr["cam"], prev or fr["cam"], keep, fr["moved"]), k5, fp[2], acc[(t + 1) & 1], None, acc[t & 1], None)
            ctx.traa_motion_blur(p, fp[2], acc[t & 1], k5, out)
            keep, prev = 1.0, fr["cam"]
            assert chain.download(7).tobytes() == acc[t & 1].download().tobytes(), (kw, t, "TRAA accumulated plane")
            got = chain.download(6)
            assert got.tobytes() == out.download().tobytes(), (kw, t, "merged TRAA + motion-blur output")
            ctx.traa_compose(acc[t & 1], out)
            blurred += int((got.view(np.uint16) != out.download().view(np.uint16)).any(-1).sum())
            for q in fp:
                q.free()
        assert blurred > 0  # the stage changed pixels K9 alone would have written
    finally:
        if chain is not None:
            chain.close()
        for q in planes:
            q.free()
        ctx.close()


@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
def test_ao_chain_with_the_stage_equals_the_effects(built, horizon):
    """5 moving frames: the AO chain with the tail and the stage writes the bytes of the AO effect, TRAAEffect.update and
    EffectPass(camera, traaEffect, motionBlurEffect) over the K7 plane, with K6 and with K6h"""
    W, H = 96, 64
    inp = ch.make_inputs(W, H, 5)
    opts = {"blueNoiseStart": 777, "iterations": 1}
    ctx = engine.Context(0, inp.blue)
    try:
        comp = Composer(ctx, W, H)
        cam, vel = Cam(inp.frames[0]["cam"]), VelocityPass()
        sc = Scene(ctx, inp.frames[0], None)
        fx = (effects.HorizonAOEffect if horizon else effects.HBAOEffect)(comp, cam, sc, opts)
        traa = _new_traa_effect(comp, cam, vel, None)
        mbfx, twin = effects.MotionBlurEffect(vel, {"intensity": 3}), effects.MotionBlurEffect(vel, {"intensity": 3})
        merged = effects.EffectPass(cam, traa, mbfx)
        chain = engine.AoChain(ctx, engine.ao_chain_options(W, H, opts, horizon=horizon))
        chain.enable_traa(abi.make_traa_tail_options())
        final, out = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
        prev = None
        for t, fr in enumerate(inp.frames):
            dt = 1 / 1000 if t % 2 == 0 else 1 / 60
            moved = effects._did_camera_move(fr["cam"], prev)
            sc.free()
            sc2 = Scene(ctx, fr, None)
            sc.depth, sc.velocity, sc.normal = sc2.depth, sc2.velocity, sc2.normal
            cam.u, vel.texture = fr["cam"], sc.velocity
            comp.inputBuffer.upload(fr["direct"])
            fx.update(None, comp.inputBuffer)
            merged.render(None, comp.outputBuffer, final, deltaTime=dt)
            chain.set_motion_blur(twin.params(comp.outputBuffer, dt))
            chain.render(fr["cam"], sc.depth, sc.velocity, sc.normal, comp.inputBuffer, out, traa_cam=fr["cam"], camera_moved=moved)
            prev = fr["cam"]
            _diff(f"frame {t} K7 plane", comp.outputBuffer.download(), chain.download(2))
            _diff(f"frame {t} TRAA accumulated", traa.temporalReprojectPass.accumulated.download(), chain.download(3))
            _diff(f"frame {t} merged TRAA + motion-blur output", final.download(), out.download())
        chain.close()
        fx.dispose()
        traa.dispose()
        for q in (final, out):
            q.free()
    finally:
        ctx.close()


def test_statuses(built):
    """status 5 = RFX_ERR_NOT_READY, 1 = RFX_ERR_INVALID_ARG (include/rfx.h)"""
    W, H = 128, 256
    inp = ch.make_inputs(W, H, 2)
    ctx = engine.Context(0, inp.blue)
    lib = ctx.lib
    p = ch.motion_blur_params(W, H)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        ssgi = engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts()))
        ao = engine.AoChain(ctx, engine.ao_chain_options(W, H, {"iterations": 1}))
        for c, kind in ((ssgi, "ssgi"), (ao, "ao")):
            fn = getattr(lib, f"rfx_{kind}_chain_set_motion_blur")
            assert fn(c.h, C.byref(p)) == 5  # the stage without the tail
            c.enable_traa()
            bad = ch.motion_blur_params(W, H, samples=0)
            assert fn(c.h, C.byref(bad)) == 1
            assert fn(c.h, C.byref(p)) == 0 and fn(c.h, None) == 0
            c.enable_traa(enable=False)  # the tail off takes the stage with it
            assert fn(c.h, C.byref(p)) == 5
        # members whose stage is on and off; a member of a group of n > 1 cannot turn the stage on or off (its values can change); the two
        # phases of a frame: a second phase 1 before the finish, and a finish with no frame waiting, are not ready
        for kind, make, fn in (("ao", lambda: engine.AoChain(ctx, engine.ao_chain_options(W, H, {"iterations": 1})), "rfx_group_attach_ao_chains_inprocess"),
                               ("ssgi", lambda: engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts())), "rfx_group_attach_chains_inprocess")):
            a, b = make(), make()
            for c in (a, b):
                c.enable_traa()
            a.set_motion_blur(p)
            st, groups = _attach(ctx, [a, b], fn)
            assert st == 1 and "motion-blur" in lib.rfx_last_error(ctx.h).decode(), kind
            for g in groups:
                lib.rfx_group_destroy(g)
            for c in (a, b):
                c.close()
        grp = parallel.InProcessAoGroup(ctx, engine.ao_chain_options(W, H, {"iterations": 1}), 2, traa=abi.make_traa_tail_options())
        assert lib.rfx_ao_chain_set_motion_blur(grp.chains[0].h, C.byref(p)) == abi.ERR_UNSUPPORTED
        assert lib.rfx_ao_chain_render_sharded_finish(grp.chains[0].h, None) == 0  # no second phase without the stage
        grp.close()
        fr = inp.frames[0]
        grp = parallel.InProcessGroup([ctx, ctx], ch.chain_options(inp, ch.Opts()), 2, traa=abi.make_traa_tail_options(), motion_blur=p)
        m = grp.chains[0]
        assert lib.rfx_ssgi_chain_set_motion_blur(m.h, None) == abi.ERR_UNSUPPORTED
        assert lib.rfx_ssgi_chain_set_motion_blur(m.h, C.byref(ch.motion_blur_params(W, H, frame=3))) == 0
        planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
        f = m._frame(abi.make_camera(fr["cam"]), *planes, fr["cam"]["position"], True)
        assert lib.rfx_ssgi_chain_render_sharded_finish(m.h, None) == 5
        assert lib.rfx_ssgi_chain_render_sharded(m.h, None, C.byref(f)) == 0
        assert lib.rfx_ssgi_chain_render_sharded(m.h, None, C.byref(f)) == 5
        assert lib.rfx_ssgi_chain_render_sharded_finish(m.h, None) == 0
        f1 = grp.chains[1]._frame(abi.make_camera(fr["cam"]), *planes, fr["cam"]["position"], True)
        assert lib.rfx_ssgi_chain_render_sharded(grp.chains[1].h, None, C.byref(f1)) == 0
        assert lib.rfx_ssgi_chain_render_sharded_finish(grp.chains[1].h, None) == 0
        ctx.sync()
        for q in planes:
            q.free()
        grp.close()
        ssgi.close()
        ao.close()
    finally:
        ctx.close()


def _moving(fr: dict, t: int) -> dict:
    """frame `fr` with a rotating velocity field (the harness's camera pans sideways: its velocities have no vertical part) that changes
    every frame; the rest of the velocity plane (packed normal, depth) is the frame's own"""
    H, W = fr["depth"].shape
    vel = np.array(fr["velocity"], copy=True)
    vel[..., :2] = ch.rotation_velocity_field(W, H, fr["depth"], 0.01 + 0.005 * t)[..., :2]
    return {**fr, "velocity": vel}


def _far_crossings(p, vel, bounds) -> int:
    """pixels whose blur taps reach more than 4 rows past their band (RFX_TRAA_TAIL_ROWS: no static halo covers them)"""
    H = vel.shape[0]
    moved, lo, hi = tap_span(p, vel)
    y = np.arange(H)[:, None].repeat(vel.shape[1], 1)
    band = np.searchsorted(np.asarray(bounds[1:-1]), y, side="right")
    b0, b1 = np.asarray(bounds)[band], np.asarray(bounds)[band + 1]
    far = (lo[..., 1] * H < b0 - 4) | (hi[..., 1] * H > b1 + 4)
    return int((moved & far).sum())


@pytest.mark.parametrize("kind", ["fast-ssgi", "ao"])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_inprocess_group_with_the_stage_is_bit_identical_to_one_chain(built, world, kind):
    """N bands on one GPU with the tail and the stage (two phases per frame, the K5 / K7 plane read on the member that owns each row),
    borders moved between frames, taps that cross band borders by far more than RFX_TRAA_TAIL_ROWS: the tail's output, the TRAA history
    and the stage's input plane equal one chain's on every frame"""
    W, H = 128, 64 * world + 112
    inp = ch.make_inputs(W, H, 5, fov=75.0)
    ctx = engine.Context(0, inp.blue)
    try:
        topt = abi.make_traa_tail_options()
        if kind == "ao":
            copt = engine.ao_chain_options(W, H, {"iterations": 1})
            single, grp_cls = engine.AoChain(ctx, copt), parallel.InProcessAoGroup
        else:
            ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
            copt = ch.chain_options(inp, ch.Opts())
            single, grp_cls = engine.SsgiChain(ctx, copt), parallel.InProcessGroup
        single.enable_traa(topt)
        single.set_motion_blur(_blur_params(0, W, H))
        grp = grp_cls(ctx, copt, world, traa=topt, motion_blur=_blur_params(0, W, H))
        b = list(grp.bounds)
        out1, outg = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
        far = 0
        for t, fr in enumerate(inp.frames):
            fr = _moving(fr, t)
            if t in (2, 4):
                grp.set_bounds([0] + [x + (16 if t == 2 else -8) for x in b[1:-1]] + [H])
            p = _blur_params(t, W, H)
            single.set_motion_blur(p)
            grp.set_motion_blur(p)
            far += _far_crossings(p, fr["velocity"], grp.bounds)
            if kind == "ao":
                d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
                single.render(fr["cam"], d, v, None, i, out1, traa_cam=fr["cam"], camera_moved=fr["moved"])
                grp.render(fr["cam"], d, v, None, i, outg, traa_cam=fr["cam"], camera_moved=fr["moved"])
                _diff(f"world {world} frame {t} output", out1.download(), outg.download())
                outs, planes = (2, 3), (d, v, i)
            else:
                planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
                cam = abi.make_camera(fr["cam"])
                single.render(cam, *planes, fr["cam"]["position"], fr["moved"])
                grp.render(cam, *planes, fr["cam"]["position"], fr["moved"])
                outs = (0, 6, 7)
            for which in outs:
                _diff(f"world {world} frame {t} output {which} bounds {grp._last_bounds}", single.download(which), grp.download(which))
            for q in planes:
                q.free()
        assert far > 0, "no tap crosses a band border by more than 4 rows: the inputs do not exercise the in-frame barrier"
        grp.close()
        single.close()
        for q in (out1, outg):
            q.free()
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
        W, H = case["w"], case["h"]
        inp = ch.make_inputs(W, H, case["frames"], fov=75.0)
        ctx = engine.Context(rank, inp.blue)
        sh = parallel.ShardedAoChain(ctx, engine.ao_chain_options(W, H, {"iterations": 1}), rebalance_every=1, rebalance_lag=1,
                                     traa=abi.make_traa_tail_options(), motion_blur=_blur_params(0, W, H))
        assert sh.uses_peer_reads == (case.get("exchange") != "allgather")
        rows = []
        for t, fr in enumerate(inp.frames):
            fr = _moving(fr, t)
            sh.set_motion_blur(_blur_params(t, W, H))
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            out = ctx.alloc(abi.FMT_RGBA16F, W, H)
            sh.render(fr["cam"], d, v, None, i, out, traa_cam=fr["cam"], camera_moved=fr["moved"])
            b0, b1 = sh.band_of_last_frame
            got = {w: sh.chain.download(w)[b0:b1].tobytes() for w in (2, 3)}
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
@pytest.mark.parametrize("exchange", [None, "allgather"])
def test_two_gpu_group_with_the_stage_equals_one_gpu(built, exchange):
    """Two processes (peer reads, or the replicated fallback), borders that move every frame: each rank's rows of the AO chain's K7 plane,
    TRAA history and merged output equal one GPU's"""
    import torch.multiprocessing as mp

    case = dict(w=256, h=256, frames=4, exchange=exchange)
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
    W, H = case["w"], case["h"]
    inp = ch.make_inputs(W, H, case["frames"], fov=75.0)
    ctx = engine.Context(0, inp.blue)
    try:
        single = engine.AoChain(ctx, engine.ao_chain_options(W, H, {"iterations": 1}))
        single.enable_traa()
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        for t, fr in enumerate(inp.frames):
            fr = _moving(fr, t)
            single.set_motion_blur(_blur_params(t, W, H))
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            single.render(fr["cam"], d, v, None, i, out, traa_cam=fr["cam"], camera_moved=fr["moved"])
            want = {w: single.download(w) for w in (2, 3)}
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
