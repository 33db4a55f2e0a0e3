"""The native AO chain (rfx_ao_chain_*) on the GPU: byte for byte the per-pass HBAOEffect / HorizonAOEffect over moving-camera frames, and
its row-sharded groups byte for byte one chain, with moving band borders, after solo frames, across two processes; and the refusals."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

import ao_harness as ao
import chain_harness as ch
from realism_effects_b200 import abi, effects, engine, parallel

pytestmark = pytest.mark.gpu

HORIZON_SMALL = {"directions": 4, "steps": 8}  # keeps the K6h grid quick at test sizes


class Scene:
    def __init__(self, ctx, fr, normal=None):
        self.depth, self.velocity = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"])
        self.normal = None if normal is None else ctx.upload(normal)

    def free(self):
        for p in (self.depth, self.velocity, self.normal):
            if p is not None:
                p.free()


class Composer:
    def __init__(self, ctx, w, h):
        self.ctx, self.width, self.height = ctx, w, h
        self.inputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)
        self.outputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)


class Cam:
    def __init__(self, u):
        self.u = u

    def uniforms(self):
        return self.u


def _diff(name, a, b):
    if a.tobytes() != b.tobytes():
        rows = np.nonzero((a.view(np.uint8).reshape(a.shape[0], -1) != b.view(np.uint8).reshape(b.shape[0], -1)).any(1))[0]
        raise AssertionError(f"{name}: rows {rows[0]}..{rows[-1]} differ ({len(rows)} rows)")


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "exact"])
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("use_normal", [False, True], ids=["depth-normal", "normal-plane"])
@pytest.mark.parametrize("iterations", [0, 1, 2])
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
def test_ao_chain_equals_the_effect(built, horizon, iterations, use_normal, scale, fast):
    """AO target, denoised plane and composed output of AoChain equal HBAOEffect / HorizonAOEffect byte for byte over 5 moving frames"""
    W, H = 96, 64
    inp = ch.make_inputs(W, H, 5)
    opts = {"blueNoiseStart": 777, "resolutionScale": scale, "useNormalPass": use_normal, "iterations": iterations, **(HORIZON_SMALL if horizon else {})}
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast)
        comp = Composer(ctx, W, H)
        cam = Cam(inp.frames[0]["cam"])
        normals = [ao.view_normal_plane(W, H, t, fr["cam"]) if use_normal else None for t, fr in enumerate(inp.frames)]
        sc = Scene(ctx, inp.frames[0], normals[0])
        fx = (effects.HorizonAOEffect if horizon else effects.HBAOEffect)(comp, cam, sc, opts)
        chain = engine.AoChain(ctx, engine.ao_chain_options(W, H, opts, horizon=horizon))
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        for t, fr in enumerate(inp.frames):
            sc.free()
            sc2 = Scene(ctx, fr, normals[t])
            sc.depth, sc.velocity, sc.normal = sc2.depth, sc2.velocity, sc2.normal
            fx._normal = sc.normal if use_normal else None
            cam.u = fr["cam"]
            comp.inputBuffer.upload(fr["direct"])
            fx.update(None, comp.inputBuffer)
            chain.render(fr["cam"], sc.depth, sc.velocity, sc.normal, comp.inputBuffer, out)
            _diff(f"frame {t} AO target", fx.aoTarget.download(), chain.download(0))
            _diff(f"frame {t} denoised", fx.texture.download(), chain.download(1))
            _diff(f"frame {t} composed", comp.outputBuffer.download(), out.download())
        chain.close()
        fx.dispose()
    finally:
        ctx.close()


def test_set_options_follows_the_effect_setters(built):
    """iterations, radius and a phi set between frames; a phi set to 0 is clamped to 1e-4 as HBAOEffect's setter does"""
    W, H = 96, 64
    inp = ch.make_inputs(W, H, 4)
    ctx = engine.Context(0, inp.blue)
    try:
        comp = Composer(ctx, W, H)
        cam = Cam(inp.frames[0]["cam"])
        sc = Scene(ctx, inp.frames[0])
        fx = effects.HBAOEffect(comp, cam, sc, {"lumaPhi": 0})
        o = {"lumaPhi": 0}
        chain = engine.AoChain(ctx, engine.ao_chain_options(W, H, o))
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        changes = [{}, {"iterations": 2, "radius": 5}, {"lumaPhi": 1e-5, "depthPhi": 0.0}, {"normalPhi": 7}]
        for t, fr in enumerate(inp.frames):
            for k, v in changes[t].items():
                setattr(fx, k, v)
            o.update(changes[t])
            chain.set_options(engine.ao_chain_options(W, H, o))
            sc.depth, sc.velocity = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"])
            cam.u = fr["cam"]
            comp.inputBuffer.upload(fr["direct"])
            fx.update(None, comp.inputBuffer)
            chain.render(fr["cam"], sc.depth, sc.velocity, None, comp.inputBuffer, out)
            _diff(f"frame {t} denoised", fx.texture.download(), chain.download(1))
            _diff(f"frame {t} composed", comp.outputBuffer.download(), out.download())
        with pytest.raises(abi.RfxError, match="algorithm"):
            chain.set_options(engine.ao_chain_options(W, H, o, horizon=True))
        with pytest.raises(abi.RfxError, match="resolution_scale"):
            chain.set_options(engine.ao_chain_options(W, H, {**o, "resolutionScale": 0.5}))
        # reset: back to a new chain's state (cleared planes, counters from their starts)
        chain.reset()
        fresh = engine.AoChain(ctx, engine.ao_chain_options(W, H, o))
        fr = inp.frames[0]
        for c in (chain, fresh):
            c.render(fr["cam"], sc.depth, sc.velocity)
        _diff("after reset", fresh.download(1), chain.download(1))
        fresh.close()
        chain.close()
    finally:
        ctx.close()


def _group_scene(world, frames):
    W, H = 320, 64 * world + 112
    inp = ch.make_inputs(W, H, frames, fov=75.0)
    bg = inp.frames[0]["depth"] == 1.0
    assert 0.15 < bg.mean() < 0.7
    return W, H, inp, bg


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "exact"])
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
@pytest.mark.parametrize("world", [2, 3, 4, 5, 8])
def test_inprocess_group_is_bit_identical_to_one_chain(built, world, horizon, fast):
    """N bands on one GPU; the wide-FOV scene whose sky silhouette crosses the borders; borders moved down at frame 2 and up at frame 4,
    so rows change owner and kept texels come from another member.  Odd N use the normal plane."""
    W, H, inp, bg = _group_scene(world, 5)
    use_normal = world % 2 == 1
    opts = {"iterations": 2, "useNormalPass": use_normal, **(HORIZON_SMALL if horizon else {})}
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_fast_math(fast)
        copt = engine.ao_chain_options(W, H, opts, horizon=horizon)
        single = engine.AoChain(ctx, copt)
        grp = parallel.InProcessAoGroup(ctx, copt, world)
        b = list(grp.bounds)
        if world >= 3:
            assert any(0.0 < bg[max(0, x - 20):x + 20].mean() < 1.0 for x in b[1:-1])
        out1, outg = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
        for t, fr in enumerate(inp.frames):
            if t == 2:
                grp.set_bounds([0] + [x + 16 for x in b[1:-1]] + [H])
            if t == 4:
                grp.set_bounds([0] + [x - 16 for x in b[1:-1]] + [H])
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            n = ctx.upload(ao.view_normal_plane(W, H, t, fr["cam"])) if use_normal else None
            single.render(fr["cam"], d, v, n, i, out1)
            grp.render(fr["cam"], d, v, n, i, outg)
            for which in (0, 1):
                _diff(f"world {world} frame {t} output {which} bounds {grp._last_bounds}", single.download(which), grp.download(which))
            _diff(f"world {world} frame {t} composed", out1.download(), outg.download())
            for p in (d, v, i, n):
                if p is not None:
                    p.free()
        grp.close()
        single.close()
    finally:
        ctx.close()


def _attach(ctx, chains, fn="rfx_group_attach_ao_chains_inprocess"):
    lib, n = ctx.lib, len(chains)
    groups = []
    for r in range(n):
        g = C.c_void_p()
        ctx._chk(lib.rfx_group_create_inprocess(ctx.h, r, n, C.byref(g)))
        groups.append(g)
    ga = (C.c_void_p * n)(*[g.value for g in groups])
    ca = (C.c_void_p * n)(*[c.h.value for c in chains])
    return getattr(lib, fn)(ga, ca, n), groups


@pytest.mark.parametrize("solo", [1, 2])
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
def test_attach_after_solo_frames_continues_from_the_latest_planes(built, horizon, solo):
    """Member chains that rendered `solo` frames alone, then attached in-process, render on from their latest planes; after the group
    is destroyed each member still holds the group's last frame in its band"""
    world = 3
    W, H, inp, _ = _group_scene(world, solo + 4)
    ctx = engine.Context(0, inp.blue)
    chains, groups = [], []
    try:
        copt = engine.ao_chain_options(W, H, {"iterations": 2, **(HORIZON_SMALL if horizon else {})}, horizon=horizon)
        chains = [engine.AoChain(ctx, copt) for _ in range(world + 1)]
        single, members = chains[0], chains[1:]
        lib = ctx.lib
        bounds = (C.c_uint32 * (world + 1))()
        for t, fr in enumerate(inp.frames):
            d, v = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"])
            single.render(fr["cam"], d, v)
            if t < solo:
                for m in members:
                    m.render(fr["cam"], d, v)
            else:
                if t == solo:
                    st, groups = _attach(ctx, members)
                    assert st == abi.RFX_OK, lib.rfx_last_error(ctx.h)
                    ctx._chk(lib.rfx_group_get_bounds(groups[0], bounds))
                    b = list(bounds)
                    moved = (C.c_uint32 * (world + 1))(*([0] + [x + 16 for x in b[1:-1]] + [H]))
                if t == solo + 2:
                    for g in groups:
                        ctx._chk(lib.rfx_group_set_bounds(g, moved))
                for m in members:
                    f = m._frame(fr["cam"], d, v)
                    ctx._chk(lib.rfx_ao_chain_render_sharded(m.h, None, C.byref(f)))
                ctx._chk(lib.rfx_group_get_last_bounds(groups[0], bounds))
                lb = list(bounds)
                for which in (0, 1):
                    want = single.download(which)
                    got = np.concatenate([m.download(which)[lb[r]:lb[r + 1]] for r, m in enumerate(members)])
                    _diff(f"solo {solo} frame {t} output {which}", want, got)
            d.free()
            v.free()
        for g in groups:
            lib.rfx_group_destroy(g)
        for r, m in enumerate(members):
            for which in (0, 1):
                _diff(f"after destroy member {r} output {which}", single.download(which)[lb[r]:lb[r + 1]], m.download(which)[lb[r]:lb[r + 1]])
    finally:
        for c in chains:
            c.close()
        ctx.close()


def test_group_refusals(built):
    W = 128
    inp = ch.make_inputs(W, 256, 1)
    ctx = engine.Context(0, inp.blue)
    lib = ctx.lib
    try:
        def status(chains, fn="rfx_group_attach_ao_chains_inprocess"):
            st, groups = _attach(ctx, chains, fn)
            msg = lib.rfx_last_error(ctx.h).decode()
            for g in groups:
                lib.rfx_group_destroy(g)
            return st, msg

        def make(h=256, **o):
            return engine.AoChain(ctx, engine.ao_chain_options(W, h, o, horizon=o.pop("horizon", False)))

        st, msg = status([make(resolutionScale=0.5), make(resolutionScale=0.5)])
        assert st == abi.ERR_UNSUPPORTED and "resolution_scale 1" in msg
        st, msg = status([make(h=192) for _ in range(4)])
        assert st == abi.ERR_UNSUPPORTED and "64 rows per rank" in msg
        st, msg = status([make(), make(horizon=True, **HORIZON_SMALL)])
        assert st == 1 and "algorithm and iterations" in msg
        st, msg = status([make(), make(iterations=2)])
        assert st == 1 and "algorithm and iterations" in msg
        # an SSGI chain and an AO chain in one group
        full = ch.make_inputs(W, 256, 1)
        ctx.set_env(full.env_map, full.env_marginal, full.env_conditional, full.env_total)
        ssgi = [engine.SsgiChain(ctx, ch.chain_options(full, ch.Opts())) for _ in range(2)]
        st, groups = _attach(ctx, ssgi, "rfx_group_attach_chains_inprocess")
        assert st == abi.RFX_OK
        aoc = [make(), make()]
        ga = (C.c_void_p * 2)(*[g.value for g in groups])
        ca = (C.c_void_p * 2)(*[c.h.value for c in aoc])
        assert lib.rfx_group_attach_ao_chains_inprocess(ga, ca, 2) == 1
        assert "cannot share a group" in lib.rfx_last_error(ctx.h).decode()
        assert lib.rfx_group_attach_ao_chain(groups[0], aoc[0].h) == 1
        assert "cannot share a group" in lib.rfx_last_error(ctx.h).decode()
        for g in groups:
            lib.rfx_group_destroy(g)
        # a chain alone takes no sharded frame
        c = make()
        f = c._frame(inp.frames[0]["cam"], ctx.upload(inp.frames[0]["depth"]), ctx.upload(inp.frames[0]["velocity"]))
        assert lib.rfx_ao_chain_render_sharded(c.h, None, C.byref(f)) == 5
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
        sh = parallel.ShardedAoChain(ctx, engine.ao_chain_options(case["w"], case["h"], case["opts"], horizon=case["horizon"]), rebalance_every=1,
                                     rebalance_lag=1)
        assert sh.uses_peer_reads == (case.get("exchange") != "allgather")
        rows = []
        for fr in inp.frames:
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            out = ctx.alloc(abi.FMT_RGBA16F, case["w"], case["h"])
            sh.render(fr["cam"], d, v, None, i, out)
            b0, b1 = sh.band_of_last_frame
            got = {w: sh.chain.download(w)[b0:b1].tobytes() for w in (0, 1)}
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
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
def test_two_gpu_group_equals_one_gpu(built, horizon, exchange):
    """Two processes with cost-driven borders that move every frame: each rank's rows equal one GPU's chain byte for byte."""
    import torch.multiprocessing as mp

    case = dict(w=256, h=256, frames=4, exchange=exchange, horizon=horizon, opts={"iterations": 1, **(HORIZON_SMALL if horizon else {})})
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
        single = engine.AoChain(ctx, engine.ao_chain_options(case["w"], case["h"], case["opts"], horizon=horizon))
        out = ctx.alloc(abi.FMT_RGBA16F, case["w"], case["h"])
        for t, fr in enumerate(inp.frames):
            d, v, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
            single.render(fr["cam"], d, v, None, i, out)
            want = {0: single.download(0), 1: single.download(1), "out": out.download()}
            for rank in range(2):
                (b0, b1), got = res[rank][t]
                for w, data in got.items():
                    assert data == want[w][b0:b1].tobytes(), (exchange, t, rank, w)
            for p in (d, v, i):
                p.free()
        single.close()
    finally:
        ctx.close()
