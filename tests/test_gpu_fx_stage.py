"""The cosmetic stage of the TRAA tail on the GPU (rfx_*_chain_set_effects): every frame of a moving-camera run is byte for byte the tail's
image followed by rfx_effects_launch with the same values, on the fast SSGI chain, the per-pass chain (SSR, full_temporal) and both AO
algorithms, with and without the motion-blur stage; the stage's input output equals the tail's output of the chain without the stage; the
AO host paths download the stage's image; in-process groups of 2 to 8 bands with moving borders equal one chain; every new status."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

import chain_harness as ch
from realism_effects_b200 import abi, engine, parallel
from test_gpu_ao_chain import _diff
from test_gpu_motion_blur_tail import _blur_params, _moving

pytestmark = pytest.mark.gpu

S, L, G, SP = abi.FX_SHARPNESS, abi.FX_LENS_DISTORTION, abi.FX_GRADUAL_BACKGROUND, abi.FX_SPARKLE
NOT_READY, INVALID_ARG = 5, 1  # include/rfx.h
# name -> (effect ids in order, values): each effect alone, the demo's SharpnessEffect({ sharpness: 0.75 }), all four in two orders, and a
# strong pincushion LensDistortion whose taps reach across several bands
FX = {
    "sharpness": ([S], dict(sharpness=1.0)),
    "lens": ([L], dict()),
    "gradual": ([G], dict(background_color=(0.2, 0.4, 0.9), max_distance=2.0)),
    "sparkle": ([SP], dict(spread=0.3, intensity=4.0)),
    "demo-sharpness-0.75": ([S], dict(sharpness=0.75)),
    "all-lens-first": ([L, S, G, SP], dict(sharpness=0.5, alphax=0.1, alphay=-0.2, aberration=2.0, background_color=(0.5, 0.1, 0.1), spread=0.3)),
    "all-lens-last": ([SP, G, S, L], dict(sharpness=0.5, alphax=0.1, alphay=-0.2, aberration=2.0, background_color=(0.5, 0.1, 0.1), spread=0.3)),
    "strong-lens": ([L, S], dict(sharpness=0.75, alphax=0.3, alphay=0.3)),
}
CHANGES = ("sharpness", "lens", "demo-sharpness-0.75", "all-lens-first", "all-lens-last", "strong-lens")  # configurations that must change pixels


def fx_params(name: str, cam_u: dict) -> abi.EffectsParams:
    ids, kw = FX[name]
    return abi.make_effects_params(cam_u, ids, **kw)


@pytest.mark.parametrize("blur", [False, True], ids=["tail", "tail+motion-blur"])
@pytest.mark.parametrize("name", list(FX), ids=str)
@pytest.mark.parametrize("kw", [dict(), dict(mode=abi.MODE_SSR, denoise_mode=1)], ids=["fast-ssgi", "ssr-full_temporal"])
def test_ssgi_chain_with_the_stage_equals_the_tail_then_the_effects(built, kw, name, blur):
    """5 moving frames: output 8 (the stage's input) == output 6 of the same chain without the stage, and output 6 == rfx_effects_launch
    over that image with the frame's depth and velocity, byte for byte; the TRAA history is untouched by the stage"""
    W, H = 160, 96
    inp = ch.make_inputs(W, H, 5)
    ctx = engine.Context(0, inp.blue)
    chains, planes = [], []
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        chains = [engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts(**kw))) for _ in range(2)]
        staged, plain = chains
        for c in chains:
            c.enable_traa(abi.make_traa_tail_options())
        ref = ctx.alloc(abi.FMT_RGBA16F, W, H)
        planes.append(ref)
        changed = 0
        for t, fr in enumerate(inp.frames):
            fp = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            p = fx_params(name, fr["cam"])
            staged.set_effects(p)
            for c in chains:
                if blur:
                    c.set_motion_blur(_blur_params(t, W, H))
                c.render(abi.make_camera(fr["cam"]), *fp, fr["cam"]["position"], fr["moved"])
            tail = plain.download(6)
            _diff(f"{name} frame {t} stage input", tail, staged.download(8))
            _diff(f"{name} frame {t} TRAA history", plain.download(7), staged.download(7))
            ctx.effects(p, plain.output(6), fp[0], fp[2], ref)
            got = staged.download(6)
            _diff(f"{name} frame {t} stage output", ref.download(), got)
            changed += int((got.view(np.uint16) != tail.view(np.uint16)).any(-1).sum())
            for q in fp:
                q.free()
        assert changed > 0 or name not in CHANGES
    finally:
        for c in chains:
            c.close()
        for q in planes:
            q.free()
        ctx.close()


def test_the_stage_turns_on_and_off_between_frames(built):
    """fast SSGI chain, 6 frames with the stage on in frames 1, 2 and 4 (values changing): output 6 is the tail's image while the stage is off,
    the stage's while it is on, and the TRAA tail never notices"""
    W, H = 160, 96
    inp = ch.make_inputs(W, H, 6)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        staged, plain = (engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts())) for _ in range(2))
        for c in (staged, plain):
            c.enable_traa(abi.make_traa_tail_options())
        ref = ctx.alloc(abi.FMT_RGBA16F, W, H)
        names = [None, "demo-sharpness-0.75", "all-lens-first", None, "lens", None]
        for t, fr in enumerate(inp.frames):
            fp = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            p = fx_params(names[t], fr["cam"]) if names[t] else None
            staged.set_effects(p)
            for c in (staged, plain):
                c.render(abi.make_camera(fr["cam"]), *fp, fr["cam"]["position"], fr["moved"])
            if p is None:
                _diff(f"frame {t} stage off", plain.download(6), staged.download(6))
                assert ctx.lib.rfx_ssgi_chain_output(staged.h, 8, C.byref(abi.Plane())) == NOT_READY
            else:
                ctx.effects(p, plain.output(6), fp[0], fp[2], ref)
                _diff(f"frame {t} stage on", ref.download(), staged.download(6))
            _diff(f"frame {t} TRAA history", plain.download(7), staged.download(7))
            for q in fp:
                q.free()
        ref.free()
        staged.close()
        plain.close()
    finally:
        ctx.close()


@pytest.mark.parametrize("blur", [False, True], ids=["tail", "tail+motion-blur"])
@pytest.mark.parametrize("name", ["demo-sharpness-0.75", "lens", "gradual", "sparkle", "all-lens-first", "all-lens-last"], ids=str)
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
def test_ao_chain_with_the_stage_equals_the_tail_then_the_effects(built, horizon, name, blur):
    """5 moving frames: output 4 (the stage's input) == frame->output of the chain without the stage, and frame->output == rfx_effects_launch
    over it; render_host and pipelined submit_host / wait_host(1) download the same bytes as the device-plane path"""
    W, H = 96, 64
    inp = ch.make_inputs(W, H, 5)
    opts = {"blueNoiseStart": 777, "iterations": 1}
    ctx = engine.Context(0, inp.blue)
    try:
        chains = [engine.AoChain(ctx, engine.ao_chain_options(W, H, opts, horizon=horizon)) for _ in range(4)]
        staged, plain, host, piped = chains
        for c in chains:
            c.enable_traa(abi.make_traa_tail_options())
        out_s, out_p, ref = (ctx.alloc(abi.FMT_RGBA16F, W, H) for _ in range(3))
        frames = [{k: np.ascontiguousarray(v) if isinstance(v, np.ndarray) else v for k, v in fr.items()} for fr in inp.frames]
        host_out = [np.zeros((H, W, 4), np.float16) for _ in frames]
        piped_out = [np.zeros((H, W, 4), np.float16) for _ in frames]
        hfs = []
        want = []
        for t, fr in enumerate(frames):
            p = fx_params(name, fr["cam"])
            for c in (staged, host, piped):
                c.set_effects(p)
            if blur:
                for c in chains:
                    c.set_motion_blur(_blur_params(t, W, H))
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            staged.render(fr["cam"], d, v, None, i, out_s, traa_cam=fr["cam"], camera_moved=fr["moved"])
            plain.render(fr["cam"], d, v, None, i, out_p, traa_cam=fr["cam"], camera_moved=fr["moved"])
            _diff(f"{name} frame {t} stage input", out_p.download(), staged.download(4))
            ctx.effects(p, out_p, d, v, ref)
            want.append(ref.download())
            _diff(f"{name} frame {t} stage output", want[-1], out_s.download())
            host.render_host(host.host_frame(fr["cam"], fr["depth"], fr["velocity"], None, fr["direct"], host_out[t], None, traa_cam=fr["cam"],
                                             camera_moved=fr["moved"]))
            _diff(f"{name} frame {t} render_host", want[-1], host_out[t])
            hfs.append(piped.host_frame(fr["cam"], fr["depth"], fr["velocity"], None, fr["direct"], piped_out[t], None, traa_cam=fr["cam"],
                                        camera_moved=fr["moved"]))
            piped.submit_host(hfs[-1])
            piped.wait_host(1)
            for q in (d, v, i):
                q.free()
        piped.wait_host(0)
        for t in range(len(frames)):
            _diff(f"{name} frame {t} submit_host", want[t], piped_out[t])
        for c in chains:
            c.close()
        for q in (out_s, out_p, ref):
            q.free()
    finally:
        ctx.close()


def test_statuses(built):
    """NOT_READY without the tail, for output 8 / AO output 4 without the stage and between the phases of a split frame; INVALID_ARG for a
    bad effect list; enable_traa(NULL) takes the stage with the tail; a group member may turn the stage on and off"""
    W, H = 128, 256
    inp = ch.make_inputs(W, H, 2)
    ctx = engine.Context(0, inp.blue)
    lib = ctx.lib
    fr = inp.frames[0]
    p = fx_params("demo-sharpness-0.75", fr["cam"])
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        ssgi = engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts()))
        ao = engine.AoChain(ctx, engine.ao_chain_options(W, H, {"iterations": 1}))
        for c, kind, stage_out in ((ssgi, "ssgi", 8), (ao, "ao", 4)):
            fn = getattr(lib, f"rfx_{kind}_chain_set_effects")
            out = getattr(lib, f"rfx_{kind}_chain_output")
            assert fn(c.h, C.byref(p)) == NOT_READY and fn(c.h, None) == NOT_READY  # the stage without the tail
            c.enable_traa()
            bad = fx_params("sharpness", fr["cam"])
            bad.n_effects = 0
            assert fn(c.h, C.byref(bad)) == INVALID_ARG
            bad.n_effects = 5
            assert fn(c.h, C.byref(bad)) == INVALID_ARG
            bad.n_effects, bad.effects[0] = 1, 7
            assert fn(c.h, C.byref(bad)) == INVALID_ARG
            assert out(c.h, stage_out, C.byref(abi.Plane())) == NOT_READY
            assert fn(c.h, C.byref(p)) == 0 and out(c.h, stage_out, C.byref(abi.Plane())) == 0
            assert fn(c.h, None) == 0 and out(c.h, stage_out, C.byref(abi.Plane())) == NOT_READY
            assert fn(c.h, C.byref(p)) == 0
            c.enable_traa(enable=False)  # the tail off takes the stage with it
            assert out(c.h, stage_out, C.byref(abi.Plane())) == NOT_READY
            c.enable_traa()
            assert out(c.h, stage_out, C.byref(abi.Plane())) == NOT_READY
        assert lib.rfx_ssgi_chain_output(ssgi.h, 9, C.byref(abi.Plane())) == INVALID_ARG
        # a group member: the stage may come and go between frames, not between the two phases of a split frame
        grp = parallel.InProcessGroup([ctx, ctx], ch.chain_options(inp, ch.Opts()), 2, traa=abi.make_traa_tail_options(),
                                      motion_blur=ch.motion_blur_params(W, H))
        m = grp.chains[0]
        assert lib.rfx_ssgi_chain_set_effects(m.h, C.byref(p)) == 0 and lib.rfx_ssgi_chain_set_effects(m.h, None) == 0
        planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
        f = m._frame(abi.make_camera(fr["cam"]), *planes, fr["cam"]["position"], True)
        assert lib.rfx_ssgi_chain_render_sharded(m.h, None, C.byref(f)) == 0
        assert lib.rfx_ssgi_chain_set_effects(m.h, C.byref(p)) == NOT_READY
        assert lib.rfx_ssgi_chain_render_sharded_finish(m.h, None) == 0
        assert lib.rfx_ssgi_chain_set_effects(m.h, C.byref(p)) == 0
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


@pytest.mark.parametrize("blur", [False, True], ids=["tail", "tail+motion-blur"])
@pytest.mark.parametrize("name", ["demo-sharpness-0.75", "strong-lens"], ids=str)
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("kind", ["fast-ssgi", "ao"])
def test_inprocess_group_with_the_stage_is_bit_identical_to_one_chain(built, kind, world, name, blur):
    """N bands on one GPU, borders moved between frames, the stage off in frame 3: the frame's final image, the stage's input and the TRAA
    history equal one chain's on every frame (with the strong lens the stage's rows of a band reach across several bands)"""
    W, H = 128, 64 * world + 112
    inp = ch.make_inputs(W, H, 5, fov=75.0)
    ctx = engine.Context(0, inp.blue)
    try:
        topt = abi.make_traa_tail_options()
        mb = _blur_params(0, W, H) if blur else None
        if kind == "ao":
            copt = engine.ao_chain_options(W, H, {"iterations": 1})
            single, grp_cls = engine.AoChain(ctx, copt), parallel.InProcessAoGroup
        else:
            ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
            copt = ch.chain_options(inp, ch.Opts())
            single, grp_cls = engine.SsgiChain(ctx, copt), parallel.InProcessGroup
        single.enable_traa(topt)
        if blur:
            single.set_motion_blur(mb)
        grp = grp_cls(ctx, copt, world, traa=topt, motion_blur=mb)
        b = list(grp.bounds)
        out1, outg = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
        reach = 0
        for t, fr in enumerate(inp.frames):
            fr = _moving(fr, t)
            if t in (2, 4):
                grp.set_bounds([0] + [x + (16 if t == 2 else -8) for x in b[1:-1]] + [H])
            p = fx_params(name, fr["cam"]) if t != 3 else None
            single.set_effects(p)
            grp.set_effects(p)
            if blur:
                single.set_motion_blur(_blur_params(t, W, H))
                grp.set_motion_blur(_blur_params(t, W, H))
            if p is not None:
                bd = grp.bounds
                ids, kw = FX[name]
                for r in range(world):
                    a, e = parallel.fx_stage_rows(W, H, (bd[r], bd[r + 1]), ids, kw.get("alphax", -0.05), kw.get("alphay", -0.05), kw.get("aberration", 1.0))
                    reach = max(reach, sum(1 for q in range(world) if q != r and a < bd[q + 1] and bd[q] < e))
            if kind == "ao":
                d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
                single.render(fr["cam"], d, v, None, i, out1, traa_cam=fr["cam"], camera_moved=fr["moved"])
                grp.render(fr["cam"], d, v, None, i, outg, traa_cam=fr["cam"], camera_moved=fr["moved"])
                _diff(f"world {world} frame {t} output", out1.download(), outg.download())
                outs, planes = ((3, 4) if p is not None else (3,)), (d, v, i)
            else:
                planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
                cam = abi.make_camera(fr["cam"])
                single.render(cam, *planes, fr["cam"]["position"], fr["moved"])
                grp.render(cam, *planes, fr["cam"]["position"], fr["moved"])
                outs = (6, 7, 8) if p is not None else (6, 7)
            for which in outs:
                _diff(f"world {world} frame {t} output {which} bounds {grp._last_bounds}", single.download(which), grp.download(which))
            for q in planes:
                q.free()
        if name == "strong-lens" and world >= 4:
            assert reach >= 2, "the strong lens does not reach across several bands"
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
        rows = []
        for t, fr in enumerate(inp.frames):
            fr = _moving(fr, t)
            sh.set_motion_blur(_blur_params(t, W, H))
            sh.set_effects(fx_params("strong-lens", fr["cam"]))
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            out = ctx.alloc(abi.FMT_RGBA16F, W, H)
            sh.render(fr["cam"], d, v, None, i, out, traa_cam=fr["cam"], camera_moved=fr["moved"])
            b0, b1 = sh.band_of_last_frame
            got = {w: sh.chain.download(w)[b0:b1].tobytes() for w in (3, 4)}
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
    """Two processes (peer reads, or the replicated fallback), borders that move every frame, the motion-blur stage and a strong lens: each
    rank's rows of the AO chain's frame output, stage input and TRAA history equal one GPU's"""
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
            single.set_effects(fx_params("strong-lens", fr["cam"]))
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            single.render(fr["cam"], d, v, None, i, out, traa_cam=fr["cam"], camera_moved=fr["moved"])
            want = {w: single.download(w) for w in (3, 4)}
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
