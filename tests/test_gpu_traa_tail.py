"""GPU tests of the chain's TRAA frame tail (rfx_ssgi_chain_enable_traa): K5 ssgi_compose -> TRAA (K2 with textureCount 1, inputType
"diffuse") -> K9 traa_compose rendered by the chain after K4.  The fast chain's fused kernel must write the bytes of the three per-pass
launches, turning the tail on must not change outputs 0..5, the tail must follow the oracle (the passes pinned to the reference shaders),
and a row-sharded group with the tail must equal one chain byte for byte."""
import os
import socket

import numpy as np
import pytest
import torch

import chain_harness as ch
from realism_effects_b200 import abi
from test_compose_options_cpu import K5_CASES
from test_march_options_cpu import make_inputs

pytestmark = pytest.mark.gpu


def _traa_params(opts, cam_u, prev_u, keep, moved):
    p = ch.traa_temporal_params(abi.make_camera(cam_u), cam_u["position"], prev_u, keep)
    p.max_blend, p.neighborhood_clamp_intensity, p.confidence_power, p.log_transform = opts.max_blend, opts.neighborhood_clamp_intensity, opts.confidence_power, opts.log_transform
    p.full_accumulate = int(bool(opts.full_accumulate) and not moved)
    return p


def _options(fog, cam_u):
    return abi.make_traa_tail_options(compose=ch.fog_params(cam_u, exp2=False) if fog else None)


def _tail_equals_per_pass_sequence(ctx, inp, o, topt, name, reset_at=None, with_plain=False):
    """Renders inp.frames with the fast chain's fused tail; every frame, outputs 6 / 7 == ssgi_compose -> temporal_reproject (TRAA form,
    RGBA16F history, LINEAR) -> traa_compose launched one by one on the chain's own `composed`, byte for byte.  reset_at: the frame
    before which the chain is reset.  with_plain: a chain without the tail runs alongside, and outputs 0..5 must be byte-identical.
    Returns the last frame's output 6."""
    from realism_effects_b200 import engine

    W, H = inp.width, inp.height
    copt = ch.chain_options(inp, o)
    chain = engine.SsgiChain(ctx, copt)
    plain = engine.SsgiChain(ctx, copt) if with_plain else None
    k5, out = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
    acc = [ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)]
    try:
        chain.enable_traa(topt)
        keep, prev = 0.0, None
        for t, fr in enumerate(inp.frames):
            if t == reset_at:
                chain.reset()
                if plain is not None:
                    plain.reset()
                keep = 0.0
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            cam = abi.make_camera(fr["cam"])
            chain.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            # the per-pass sequence on the chain's own `composed`
            ctx.ssgi_compose(planes[0], chain.output(0), planes[3], k5, params=topt.compose)
            tp = _traa_params(topt, fr["cam"], prev or fr["cam"], keep, fr["moved"])
            ctx.temporal_reproject(tp, k5, planes[2], acc[(t + 1) & 1], None, acc[t & 1], None)
            ctx.traa_compose(acc[t & 1], out)
            keep, prev = 1.0, fr["cam"]
            got6, got7 = chain.download(6), chain.download(7)
            assert got7.tobytes() == acc[t & 1].download().tobytes(), (name, t, "TRAA accumulated plane")
            assert got6.tobytes() == out.download().tobytes(), (name, t, "K9 output")
            assert np.isfinite(got6).all() and (got6[..., 3] == 1).all()
            if plain is not None:
                plain.render(cam, *planes, fr["cam"]["position"], fr["moved"])
                for which in range(6):
                    assert chain.download(which).tobytes() == plain.download(which).tobytes(), (name, t, which)
            for p in planes:
                p.free()
        return got6
    finally:
        chain.close()
        if plain is not None:
            plain.close()
        for q in [k5, out] + acc:
            q.free()


@pytest.mark.parametrize("size", [(320, 192), (3840, 2160)])
@pytest.mark.parametrize("fog", [False, True])
def test_fused_tail_writes_the_bytes_of_the_per_pass_sequence(built, size, fog):
    """4 frames with history and a reset before frame 2: the fused tail writes the bytes of the per-pass sequence every frame.  At the
    small size a chain without the tail runs alongside: outputs 0..5 are byte-identical with and without it."""
    from realism_effects_b200 import engine

    W, H = size
    inp = ch.make_inputs(W, H, 4, device="cuda" if W > 1000 else "cpu")
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        got6 = _tail_equals_per_pass_sequence(ctx, inp, ch.Opts(denoise_iterations=1 if W > 1000 else 2), _options(fog, inp.frames[0]["cam"]),
                                              f"{size} fog={fog}", reset_at=2, with_plain=W < 1000)
        assert np.abs(got6[..., :3].astype(np.float32)).max() > 0.05
    finally:
        ctx.close()


@pytest.mark.parametrize("case", K5_CASES, ids=str)
def test_fused_tail_writes_the_bytes_of_the_per_pass_sequence_across_k5_options(built, case):
    """3 frames at each point of the SSGI compose grid (tests/test_compose_options_cpu.py: no fog, linear fog and FogExp2 with
    perspective and orthographic cameras, isDebug, odd sizes and a 3840x16 strip) as the tail's compose options: the fused tail
    (ctraa_kernel, which shares ssgi_compose_px with ssgi_compose_kernel) writes the bytes of the per-pass sequence every frame"""
    from realism_effects_b200 import engine

    inp = make_inputs(case.W, case.H, case.camera, frames=3)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        _tail_equals_per_pass_sequence(ctx, inp, ch.Opts(), abi.make_traa_tail_options(compose=case.params(inp.frames[0]["cam"])), str(case))
    finally:
        ctx.close()


@pytest.mark.parametrize("kw", [dict(), dict(mode=abi.MODE_SSR), dict(fast_math=False)], ids=["fast", "ssr", "exact"])
def test_tail_follows_the_oracle(built, kw):
    """The tail over 3 frames vs orc.ssgi_compose -> orc.temporal_reproject(out_half=True) -> orc.traa_compose on the ORACLE chain's
    `composed`: within the bar tests/test_gpu_effects.py uses for TRAA (<= 2e-3 of the pixels outside 1e-3).  The fast chain runs the fused
    kernel; SSR mode and fast_math off run the three per-pass launches."""
    import orc

    from realism_effects_b200 import engine

    fast = kw.pop("fast_math", True)
    o = ch.Opts(**kw)
    inp = ch.make_inputs(320, 192, 3)
    ref = ch.run_oracle_chain(inp, o, capture=("composed",), lean=True)
    topt = abi.make_traa_tail_options()
    ctx = engine.Context(0, inp.blue)
    ctx.set_fast_math(fast)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        chain = engine.SsgiChain(ctx, ch.chain_options(inp, o))
        chain.enable_traa(topt)
        hist, keep, prev = np.zeros((192, 320, 4), np.float16), 0.0, None
        for t, fr in enumerate(inp.frames):
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            chain.render(abi.make_camera(fr["cam"]), *planes, fr["cam"]["position"], fr["moved"])
            k5 = orc.ssgi_compose(fr["depth"], ref[t]["composed"], fr["direct"])
            tp = _traa_params(topt, fr["cam"], prev or fr["cam"], keep, fr["moved"])
            hist, _ = orc.temporal_reproject(tp, k5, fr["velocity"], hist, None, hist, None, out_half=True)
            keep, prev = 1.0, fr["cam"]
            c7 = ch.compare(hist, chain.download(7))
            c6 = ch.compare(orc.traa_compose(hist), chain.download(6))
            assert c7["frac_bad"] <= 2e-3 and c6["frac_bad"] <= 2e-3, (t, c7, c6)
            for p in planes:
                p.free()
        chain.close()
    finally:
        ctx.close()


@pytest.mark.parametrize("world", [2, 3, 4, 5, 8])
def test_inprocess_group_with_the_tail_is_bit_identical_to_one_chain(built, world):
    """In-process group of N bands with the tail (its K4 range widened by RFX_TRAA_TAIL_ROWS, the TRAA history read on the member that
    owns the row), the wide-FOV scene whose sky silhouette crosses the borders, borders moved at frames 2 and 4: outputs 0, 1, 4, 5, 6, 7
    equal one chain with the tail byte for byte on every frame."""
    from realism_effects_b200 import engine, parallel

    W, H = 320, 64 * world + 112
    o = ch.Opts(denoise_iterations=2)
    inp = ch.make_inputs(W, H, 5, fov=75.0)
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, o)
        topt = abi.make_traa_tail_options()
        single = engine.SsgiChain(ctx, copt)
        single.enable_traa(topt)
        grp = parallel.InProcessGroup(ctx, copt, world, traa=topt)
        b = list(grp.bounds)
        for t, fr in enumerate(inp.frames):
            if t == 2:
                grp.set_bounds([0] + [x + 16 for x in b[1:-1]] + [H])
            if t == 4:
                grp.set_bounds([0] + [x - 16 for x in b[1:-1]] + [H])
            planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            cam = abi.make_camera(fr["cam"])
            single.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            grp.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            for which in (0, 1, 4, 5, 6, 7):
                a, g = single.download(which), grp.download(which)
                if a.tobytes() != g.tobytes():
                    rows = np.nonzero((a.view(np.uint8).reshape(H, -1) != g.view(np.uint8).reshape(H, -1)).any(1))[0]
                    raise AssertionError(f"world {world} frame {t} output {which}: rows {rows[0]}..{rows[-1]} differ ({len(rows)} rows); bounds {grp._last_bounds}")
            for p in planes:
                p.free()
        grp.close()
        single.close()
    finally:
        ctx.close()


def test_tail_error_cases(built):
    import ctypes as C

    from realism_effects_b200 import engine, parallel

    o = ch.Opts()
    inp = ch.make_inputs(160, 128, 1)
    fr = inp.frames[0]
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        copt = ch.chain_options(inp, o)
        chain = engine.SsgiChain(ctx, copt)
        planes = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
        cam = abi.make_camera(fr["cam"])
        chain.render(cam, *planes, fr["cam"]["position"], fr["moved"])
        for which in (6, 7):  # outputs of the tail while it is off
            with pytest.raises(abi.RfxError, match="status 5"):
                chain.output(which)
        chain.enable_traa()
        with pytest.raises(abi.RfxError, match="status 1"):  # the tail composes over the direct light plane
            chain.render(cam, *planes[:3], None, fr["cam"]["position"], fr["moved"])
        chain.render(cam, *planes, fr["cam"]["position"], fr["moved"])
        assert chain.download(6).shape == (128, 160, 4)
        chain.enable_traa(enable=False)
        with pytest.raises(abi.RfxError, match="status 5"):
            chain.output(6)
        chain.close()
        grp = parallel.InProcessGroup(ctx, copt, 2)  # a group's peer mappings are fixed at attach time
        with pytest.raises(abi.RfxError, match="status 6"):
            grp.chains[0].enable_traa()
        grp.close()
        buf = C.create_string_buffer(abi.GROUP_ID_BYTES)
        ctx._chk(ctx.lib.rfx_group_get_unique_id(buf))
        sh = parallel.ShardedSsgiChain(ctx, copt, rank=0, world=1, unique_id=bytes(buf.raw), traa=abi.make_traa_tail_options())
        host = {k: torch.from_numpy(np.ascontiguousarray(fr[n])) for k, n in (("depth", "depth"), ("gbuffer", "gbuffer"), ("velocity", "velocity"), ("direct", "direct"))}
        with pytest.raises(abi.RfxError, match="status 6"):
            sh.submit_host(cam, host, fr["cam"]["position"], fr["moved"], torch.zeros(128 * 160 * 4))
        sh.close()
        for p in planes:
            p.free()
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
        inp = ch.make_inputs(case["w"], case["h"], case["frames"])
        ctx = engine.Context(rank, inp.blue)
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        sh = parallel.ShardedSsgiChain(ctx, ch.chain_options(inp, ch.Opts(denoise_iterations=1)), rebalance_every=1, rebalance_lag=1,
                                       traa=abi.make_traa_tail_options())
        assert sh.uses_peer_reads == (case.get("exchange") != "allgather")
        keep, rows = [], []
        for fr in inp.frames:
            pl = [ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")]
            keep.append(pl)
            sh.render(abi.make_camera(fr["cam"]), *pl, fr["cam"]["position"], fr["moved"])
            b0, b1 = sh.band_of_last_frame
            rows.append(((b0, b1), {w: sh.chain.download(w)[b0:b1].tobytes() for w in (0, 4, 5, 6, 7)}))
        q.put((rank, rows))
        sh.close()
        ctx.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("exchange", [None, "allgather"])
def test_two_gpu_group_with_the_tail_equals_one_gpu(built, exchange):
    import torch.multiprocessing as mp

    from realism_effects_b200 import engine

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
    inp = ch.make_inputs(case["w"], case["h"], case["frames"])
    ctx = engine.Context(0, inp.blue)
    try:
        ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
        single = engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts(denoise_iterations=1)))
        single.enable_traa()
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
