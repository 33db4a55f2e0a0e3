"""Row-sharded groups of the per-pass chain: SSR mode in every denoise mode, and SSGI mode in denoiseMode "full_temporal" / "temporal",
with and without the TRAA tail.  Every member's rows of every chain output must equal one chain with the same options byte for byte,
with band borders that move between frames; the configurations a group does not take are refused with a reason."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

import chain_harness as ch
from realism_effects_b200 import abi

pytestmark = pytest.mark.gpu

FULL, FULL_TEMPORAL, TEMPORAL = 0, 1, 2
CONFIGS = [  # (mode, denoise_mode, TRAA tail)
    (abi.MODE_SSR, FULL, False),
    (abi.MODE_SSR, FULL_TEMPORAL, False),
    (abi.MODE_SSR, TEMPORAL, False),
    (abi.MODE_SSGI, FULL_TEMPORAL, False),
    (abi.MODE_SSGI, TEMPORAL, False),
    (abi.MODE_SSR, FULL_TEMPORAL, True),
    (abi.MODE_SSGI, TEMPORAL, True),
]


def _outputs(mode, dm, tail):
    """chain outputs this configuration writes (0 is `composed`, or tr[0] in "temporal"; 3 and 5 are the SSGI specular planes; 4 and 5
    are the Poisson targets of "full"; 6 and 7 the TRAA tail's)"""
    out = [0, 1, 2]
    if mode == abi.MODE_SSGI:
        out.append(3)
    if dm == FULL:
        out += [4, 5] if mode == abi.MODE_SSGI else [4]
    if tail:
        out += [6, 7]
    return out


def _cfg_id(c):
    return f"{'ssgi' if c[0] == abi.MODE_SSGI else 'ssr'}-{('full', 'full_temporal', 'temporal')[c[1]]}{'-traa' if c[2] else ''}"


@pytest.mark.parametrize("world", [2, 3, 4, 5, 8])
@pytest.mark.parametrize("cfg", CONFIGS, ids=_cfg_id)
def test_inprocess_group_of_the_per_pass_chain_is_bit_identical_to_one_chain(built, cfg, world):
    """In-process group of N bands on one GPU; the wide-FOV scene whose sky silhouette (discarded pixels next to shaded ones) crosses the
    borders; borders moved down at frame 2 and up at frame 4, so rows change owner and kept texels / history come from another member."""
    from realism_effects_b200 import engine, parallel

    mode, dm, tail = cfg
    W, H = 320, 64 * world + 112
    o = ch.Opts(mode=mode, denoise_mode=dm, denoise_iterations=2)
    inp = ch.make_inputs(W, H, 5, fov=75.0)
    bg = inp.frames[0]["depth"] == 1.0
    assert 0.15 < bg.mean() < 0.7
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, o)
        topt = abi.make_traa_tail_options() if tail else None
        single = engine.SsgiChain(ctx, copt)
        if tail:
            single.enable_traa(topt)
        grp = parallel.InProcessGroup(ctx, copt, world, traa=topt)
        b = list(grp.bounds)
        if world >= 3:
            assert any(0.0 < bg[max(0, x - 20):x + 20].mean() < 1.0 for x in b[1:-1])
        for t, fr in enumerate(inp.frames):
            if t == 2:
                grp.set_bounds([0] + [x + 16 for x in b[1:-1]] + [H])
            if t == 4:
                grp.set_bounds([0] + [x - 16 for x in b[1:-1]] + [H])
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            cam = abi.make_camera(fr["cam"])
            single.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            grp.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            for which in _outputs(mode, dm, tail):
                a, g = single.download(which), grp.download(which)
                if a.tobytes() != g.tobytes():
                    rows = np.nonzero((a.view(np.uint8).reshape(H, -1) != g.view(np.uint8).reshape(H, -1)).any(1))[0]
                    raise AssertionError(f"{_cfg_id(cfg)} world {world} frame {t} output {which}: rows {rows[0]}..{rows[-1]} differ ({len(rows)} rows); "
                                         f"bounds {grp._last_bounds}")
            for p in planes:
                p.free()
        grp.close()
        single.close()
    finally:
        ctx.close()


def _attach_inprocess(ctx, chains):
    """rfx_group_attach_chains_inprocess over `chains` (one in-process group member each); returns the status and the groups"""
    lib, n = ctx.lib, len(chains)
    groups = []
    for r in range(n):
        g = C.c_void_p()
        ctx._chk(lib.rfx_group_create_inprocess(ctx.h, r, n, C.byref(g)))
        groups.append(g)
    ga = (C.c_void_p * n)(*[g.value for g in groups])
    ca = (C.c_void_p * n)(*[c.h.value if hasattr(c.h, "value") else c.h for c in chains])
    return lib.rfx_group_attach_chains_inprocess(ga, ca, n), groups


@pytest.mark.parametrize("solo", [1, 2])
@pytest.mark.parametrize("tail", [False, True], ids=["", "traa"])
@pytest.mark.parametrize("cfg", [(abi.MODE_SSGI, FULL), (abi.MODE_SSR, FULL_TEMPORAL)], ids=["fast", "ssr-full_temporal"])
def test_attach_after_solo_frames_continues_from_the_latest_planes(built, request, cfg, tail, solo):
    """Member chains that rendered `solo` frames alone, then were attached in-process, render on from their latest planes: with
    moving borders every output equals one chain byte for byte.  After the group is destroyed, each member's outputs still hold the
    group's last frame in its band."""
    from realism_effects_b200 import engine

    mode, dm = cfg
    if dm == FULL and solo % 2 == 0:
        request.applymarker(pytest.mark.xfail(strict=True, reason="the fast chain's Poisson target A is single-buffered alone: after an even "
                                              "number of solo frames the group's first frame carries A's discarded texels from buffer 1, "
                                              "which the chain never wrote"))
    world = 3
    W, H = 320, 64 * world + 112
    inp = ch.make_inputs(W, H, solo + 4, fov=75.0)
    ctx = engine.Context(0, inp.blue)
    chains, groups = [], []
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, ch.Opts(mode=mode, denoise_mode=dm, denoise_iterations=2))
        chains = [engine.SsgiChain(ctx, copt) for _ in range(world + 1)]
        if tail:
            for c in chains:
                c.enable_traa(abi.make_traa_tail_options())
        single, members = chains[0], chains[1:]
        lib, outputs = ctx.lib, _outputs(mode, dm, tail)
        bounds = (C.c_uint32 * (world + 1))()
        for t, fr in enumerate(inp.frames):
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            cam = abi.make_camera(fr["cam"])
            single.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            if t < solo:
                for c in members:
                    c.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            else:
                if t == solo:
                    st, groups = _attach_inprocess(ctx, members)
                    assert st == 0, lib.rfx_last_error(ctx.h)
                    ctx._chk(lib.rfx_group_get_bounds(groups[0], bounds))
                    b = list(bounds)
                elif t >= solo + 2:  # borders down by 16 rows, then back
                    step = 16 if t == solo + 2 else 0
                    new = (C.c_uint32 * (world + 1))(*([0] + [x + step for x in b[1:-1]] + [H]))
                    for g in groups:
                        ctx._chk(lib.rfx_group_set_bounds(g, new))
                ctx._chk(lib.rfx_group_get_bounds(groups[0], bounds))
                last = list(bounds)
                for c in members:
                    f = c._frame(cam, *planes, fr["cam"]["position"], fr["moved"])
                    ctx._chk(lib.rfx_ssgi_chain_render_sharded(c.h, None, C.byref(f)))
                ctx.sync()
                for which in outputs:
                    a = single.download(which)
                    g = np.concatenate([c.download(which)[last[r]:last[r + 1]] for r, c in enumerate(members)], axis=0)
                    if a.tobytes() != g.tobytes():
                        rows = np.nonzero((a.view(np.uint8).reshape(H, -1) != g.view(np.uint8).reshape(H, -1)).any(1))[0]
                        raise AssertionError(f"frame {t} output {which}: rows {rows[0]}..{rows[-1]} differ ({len(rows)} rows); bounds {last}")
            for p in planes:
                p.free()
        for g in groups:
            lib.rfx_group_destroy(g)
        groups = []
        for which in outputs:
            a = single.download(which)
            for r, c in enumerate(members):
                assert c.download(which)[last[r]:last[r + 1]].tobytes() == a[last[r]:last[r + 1]].tobytes(), (which, r)
    finally:
        for g in groups:
            ctx.lib.rfx_group_destroy(g)
        for c in chains:
            c.close()
        ctx.close()


def test_group_refusals(built):
    """fast_math off and resolution_scale < 1 are refused (status 6, RFX_ERR_UNSUPPORTED), members with different modes are invalid
    (status 1), and the sharded host path refuses the per-pass chain (status 6)."""
    from realism_effects_b200 import engine, parallel

    inp = ch.make_inputs(160, 128, 1)
    fr = inp.frames[0]
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        cases = [  # (options of member 0, of member 1, fast_math, expected status, message)
            (ch.Opts(mode=abi.MODE_SSR), ch.Opts(mode=abi.MODE_SSR), False, 6, "fast_math"),
            (ch.Opts(mode=abi.MODE_SSR, resolution_scale=0.5), ch.Opts(mode=abi.MODE_SSR, resolution_scale=0.5), True, 6, "resolution_scale"),
            (ch.Opts(denoise_mode=FULL_TEMPORAL), ch.Opts(denoise_mode=FULL_TEMPORAL), False, 6, "fast_math"),
            (ch.Opts(mode=abi.MODE_SSR, denoise_mode=FULL_TEMPORAL), ch.Opts(denoise_mode=FULL_TEMPORAL), True, 1, "same mode"),
            (ch.Opts(mode=abi.MODE_SSR), ch.Opts(mode=abi.MODE_SSR, denoise_mode=TEMPORAL), True, 1, "same mode"),
        ]
        for o0, o1, fast, want, msg in cases:
            ctx.set_fast_math(fast)
            chains = [engine.SsgiChain(ctx, ch.chain_options(inp, o0)), engine.SsgiChain(ctx, ch.chain_options(inp, o1))]
            st, groups = _attach_inprocess(ctx, chains)
            assert st == want, (o0, o1, fast, st)
            assert msg in ctx.lib.rfx_last_error(ctx.h).decode(), ctx.lib.rfx_last_error(ctx.h)
            for g in groups:
                ctx.lib.rfx_group_destroy(g)
            for c in chains:
                c.close()
        ctx.set_fast_math(True)
        buf = C.create_string_buffer(abi.GROUP_ID_BYTES)
        ctx._chk(ctx.lib.rfx_group_get_unique_id(buf))
        sh = parallel.ShardedSsgiChain(ctx, ch.chain_options(inp, ch.Opts(mode=abi.MODE_SSR, denoise_mode=FULL_TEMPORAL)), rank=0, world=1,
                                       unique_id=bytes(buf.raw))
        cam = abi.make_camera(fr["cam"])
        host = {k: torch.from_numpy(np.ascontiguousarray(fr[n])) for k, n in (("depth", "depth"), ("gbuffer", "gbuffer"), ("velocity", "velocity"), ("direct", "direct"))}
        with pytest.raises(abi.RfxError, match="status 6"):
            sh.submit_host(cam, host, fr["cam"]["position"], fr["moved"], torch.zeros(128 * 160 * 4))
        sh.close()
    finally:
        ctx.close()


# ---- two processes, one GPU each (rfx_group_create: CUDA-IPC peer mappings or the NCCL all-gather fallback) ------------------------------
def _worker(rank, world, port, q, case):
    import torch.distributed as dist

    from realism_effects_b200 import engine, parallel

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    if case.get("exchange"):
        os.environ["RFX_GROUP_EXCHANGE"] = case["exchange"]
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        inp = ch.make_inputs(case["w"], case["h"], case["frames"], fov=75.0)
        ctx = engine.Context(rank, inp.blue)
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        sh = parallel.ShardedSsgiChain(ctx, ch.chain_options(inp, ch.Opts(mode=case["mode"], denoise_mode=case["dm"])), rebalance_every=1, rebalance_lag=1)
        assert sh.uses_peer_reads == (case.get("exchange") != "allgather")
        keep, rows = [], []
        for fr in inp.frames:
            pl = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            keep.append(pl)
            sh.render(abi.make_camera(fr["cam"]), *pl, fr["cam"]["position"], fr["moved"])
            b0, b1 = sh.band_of_last_frame
            rows.append(((b0, b1), {w: sh.chain.download(w)[b0:b1].tobytes() for w in case["outputs"]}))
        q.put((rank, rows))
        sh.close()
        ctx.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("exchange", [None, "allgather"])
@pytest.mark.parametrize("cfg", [(abi.MODE_SSR, FULL_TEMPORAL), (abi.MODE_SSGI, TEMPORAL)], ids=["ssr-full_temporal", "ssgi-temporal"])
def test_two_gpu_group_of_the_per_pass_chain_equals_one_gpu(built, cfg, exchange):
    """Two processes with cost-driven borders that move every frame: each rank's rows equal one GPU's chain byte for byte."""
    import torch.multiprocessing as mp

    from realism_effects_b200 import engine

    mode, dm = cfg
    case = dict(w=256, h=256, frames=4, exchange=exchange, mode=mode, dm=dm, outputs=_outputs(mode, dm, False))
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
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        single = engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts(mode=mode, denoise_mode=dm)))
        for t, fr in enumerate(inp.frames):
            pl = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            single.render(abi.make_camera(fr["cam"]), *pl, fr["cam"]["position"], fr["moved"])
            for rank in range(2):
                (b0, b1), got = res[rank][t]
                for w, data in got.items():
                    assert data == single.download(w)[b0:b1].tobytes(), (exchange, t, rank, w)
            for p in pl:
                p.free()
        single.close()
    finally:
        ctx.close()
