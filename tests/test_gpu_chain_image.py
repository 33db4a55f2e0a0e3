"""The SSGI chain's compose stage on the GPU (rfx_ssgi_chain_set_compose, output 9) and the host path's image download (out_color).
Output 9 is byte for byte rfx_ssgi_compose_launch over output 0 of the same frame, in every chain configuration (the fast chain's fused
K4 epilogue with the plain and the TMA Poisson pass, and the per-pass chains), with and without fog, and with a debug view selected;
the stage changes none of outputs 0-5; render_host and pipelined submit_host / wait_host(1) download the device planes (output 9, or the
TRAA tail's output 6); in-process groups of 2 to 8 bands with moving borders equal one chain; every new status."""
import ctypes as C

import numpy as np
import pytest
import torch

import chain_harness as ch
from realism_effects_b200 import abi, engine, parallel
from test_gpu_ao_chain import _diff
from test_gpu_fx_stage import fx_params
from test_gpu_motion_blur_tail import _blur_params, _moving

pytestmark = pytest.mark.gpu

INVALID_ARG, NOT_READY = 1, 5  # include/rfx.h
IN = ("depth", "gbuffer", "velocity", "direct")
# name -> (chain options, fast_math, RFX_K3_TMA)
CONFIGS = {
    "fast-it0": (dict(denoise_iterations=0), True, "1"),
    "fast-it1": (dict(denoise_iterations=1), True, "1"),
    "fast-it2-tma": (dict(denoise_iterations=2), True, "1"),
    "fast-it2-plain": (dict(denoise_iterations=2), True, "0"),
    "ssr": (dict(mode=abi.MODE_SSR), True, "1"),
    "full_temporal": (dict(denoise_mode=abi.DENOISE_FULL_TEMPORAL), True, "1"),
    "temporal": (dict(denoise_mode=abi.DENOISE_TEMPORAL), True, "1"),
    "scale-0.5": (dict(resolution_scale=0.5), True, "1"),
    "exact": (dict(), False, "1"),
}


def compose_params(cam_u: dict, fog: str) -> abi.SsgiComposeParams:
    """K5's values for the frame's camera: no fog, three's Fog or FogExp2 (chain_harness.fog_params' values)"""
    if fog == "none":
        p = abi.SsgiComposeParams()
        p.camera_near, p.camera_far = float(cam_u["near"]), float(cam_u["far"])
    else:
        p = ch.fog_params(cam_u, fog == "exp2")
    p.perspective = int(bool(cam_u.get("perspective", True)))
    return p


def _context(inp, fast_math=True):
    ctx = engine.Context(0, inp.blue)
    ctx.set_fast_math(fast_math)
    ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    return ctx


def _run_stage(inp, opts, fast_math, fog, view=None):
    """3 frames (camera moving) on a chain with the stage and one without: per frame, output 9 against rfx_ssgi_compose_launch over output
    0 (or, with a debug view, over the view with isDebug), and outputs 0-5 against the plain chain"""
    W, H = inp.width, inp.height
    ctx = _context(inp, fast_math)
    try:
        copt = ch.chain_options(inp, ch.Opts(**opts))
        staged, plain = engine.SsgiChain(ctx, copt), engine.SsgiChain(ctx, copt)
        ref, gdbg = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA32F, W, H)
        if view is not None:
            staged.set_debug_view(view)
        for t, fr in enumerate(inp.frames):
            fp = [ctx.upload(fr[k]) for k in IN]
            p = compose_params(fr["cam"], fog)
            staged.set_compose(p)
            for c in (staged, plain):
                c.render(abi.make_camera(fr["cam"]), *fp, fr["cam"]["position"], fr["moved"])
            if view is None:
                ctx.ssgi_compose(fp[0], staged.output(0), fp[3], ref, params=p)
            else:
                q = compose_params(fr["cam"], fog)
                q.is_debug = 1
                if view == abi.DEBUG_VIEW_DEPTH:
                    v = fp[0]
                elif view >= abi.DEBUG_VIEW_GBUFFER_CHANNEL:
                    ctx.gbuffer_debug(view - abi.DEBUG_VIEW_GBUFFER_CHANNEL, fp[1], gdbg)
                    v = gdbg
                else:
                    v = staged.output(view - abi.DEBUG_VIEW_OUTPUT)
                ctx.ssgi_compose(fp[0], v, fp[3], ref, params=q)
            _diff(f"frame {t} output 9", ref.download(), staged.download(9))
            for which in range(6):
                _diff(f"frame {t} output {which}", plain.download(which), staged.download(which))
            for q_ in fp:
                q_.free()
        staged.close()
        plain.close()
        ref.free()
        gdbg.free()
    finally:
        ctx.close()


@pytest.mark.parametrize("fog", ["none", "fog", "exp2"])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_output9_is_the_compose_launch_over_output0(built, monkeypatch, config, fog):
    opts, fast_math, tma = CONFIGS[config]
    monkeypatch.setenv("RFX_K3_TMA", tma)
    _run_stage(ch.make_inputs(160, 96, 3), opts, fast_math, fog)


@pytest.mark.parametrize("config", ["fast-it1", "ssr"])
def test_output9_orthographic(built, config):
    opts, fast_math, _ = CONFIGS[config]
    _run_stage(ch.make_inputs(160, 96, 3, orthographic=True), opts, fast_math, "fog")


@pytest.mark.parametrize("view", [abi.DEBUG_VIEW_OUTPUT + 1, abi.DEBUG_VIEW_OUTPUT + 4, abi.DEBUG_VIEW_DEPTH, abi.DEBUG_VIEW_GBUFFER_CHANNEL + 2],
                         ids=["ssgiOut", "dnB0", "depth", "gbuffer-normal"])
@pytest.mark.parametrize("config", ["fast-it1", "ssr"])
def test_debug_view_through_the_stage_is_the_per_pass_isdebug_k5(built, config, view):
    opts, fast_math, _ = CONFIGS[config]
    _run_stage(ch.make_inputs(160, 96, 3), opts, fast_math, "none", view=view)


def _pinned(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


# name -> (chain options, what the frame's image is: "stage", "tail", "tail+mb", "tail+fx")
HOST_CASES = {
    "stage-fast": (dict(), "stage"), "stage-fast-it0": (dict(denoise_iterations=0), "stage"), "stage-ssr": (dict(mode=abi.MODE_SSR), "stage"),
    "stage-temporal": (dict(denoise_mode=abi.DENOISE_TEMPORAL), "stage"),
    "tail-fast": (dict(), "tail"), "tail-ssr": (dict(mode=abi.MODE_SSR), "tail"), "tail+mb-fast": (dict(), "tail+mb"), "tail+fx-fast": (dict(), "tail+fx"),
}


@pytest.mark.parametrize("composed", [False, True], ids=["image-only", "both"])
@pytest.mark.parametrize("case", list(HOST_CASES))
def test_host_paths_download_the_device_planes(built, case, composed):
    """5 moving frames on three chains: device planes, render_host, and pipelined submit_host / wait_host(1) over two alternating pinned host
    sets (a set is refilled only after the wait that releases it).  out_color == output 9 (stage) or output 6 (tail), out_composed == the
    host path's `composed`, frame for frame."""
    opts, image = HOST_CASES[case]
    inp = ch.make_inputs(160, 96, 5)
    W, H = inp.width, inp.height
    ctx = _context(inp)
    try:
        copt = ch.chain_options(inp, ch.Opts(**opts))
        dev, sync, piped = chains = [engine.SsgiChain(ctx, copt) for _ in range(3)]
        frames = [_moving(fr, t) for t, fr in enumerate(inp.frames)]
        for c in chains:
            if image == "stage":
                continue
            c.enable_traa(abi.make_traa_tail_options())
            if image == "tail+mb":
                c.set_motion_blur(_blur_params(0, W, H))
        which = 9 if image == "stage" else 6
        sets = [{k: _pinned(frames[0][k]) for k in IN} for _ in range(2)]
        outs = [(torch.zeros((H, W, 4), dtype=torch.float32).pin_memory(), torch.zeros((H, W, 4), dtype=torch.float16).pin_memory()) for _ in range(2)]
        got_sync, got_piped, want = [], [], []

        def per_frame(c, t, fr):
            if image == "stage":
                c.set_compose(compose_params(fr["cam"], "fog"))
            elif image == "tail+mb":
                c.set_motion_blur(_blur_params(t, W, H))
            elif image == "tail+fx":
                c.set_effects(fx_params("demo-sharpness-0.75", fr["cam"]))

        def host_frame(c, fr, hs, out):
            return c.host_frame(abi.make_camera(fr["cam"]), hs["depth"], hs["gbuffer"], hs["velocity"], hs["direct"], fr["cam"]["position"],
                                fr["moved"], out[0] if composed else None, out[1])

        for t, fr in enumerate(frames):
            fp = [ctx.upload(fr[k]) for k in IN]
            per_frame(dev, t, fr)
            dev.render(abi.make_camera(fr["cam"]), *fp, fr["cam"]["position"], fr["moved"])
            want.append(dev.download(which))
            for q in fp:
                q.free()
            per_frame(sync, t, fr)
            hs = {k: _pinned(fr[k]) for k in IN}
            o = (torch.zeros((H, W, 4), dtype=torch.float32), torch.zeros((H, W, 4), dtype=torch.float16))
            sync.render_host(host_frame(sync, fr, hs, o))
            got_sync.append((o[0].numpy().copy(), o[1].numpy().copy()))
            # pipelined: frame t in set t & 1
            s = t & 1
            for k in IN:
                sets[s][k].copy_(torch.from_numpy(np.ascontiguousarray(fr[k])))
            per_frame(piped, t, fr)
            piped.submit_host(host_frame(piped, fr, sets[s], outs[s]))
            piped.wait_host(1)
            if t >= 1:
                o = outs[s ^ 1]
                got_piped.append((o[0].numpy().copy(), o[1].numpy().copy()))
        piped.wait_host(0)
        o = outs[(len(frames) - 1) & 1]
        got_piped.append((o[0].numpy().copy(), o[1].numpy().copy()))
        for t in range(len(frames)):
            _diff(f"{case} frame {t} render_host out_color", want[t], got_sync[t][1])
            _diff(f"{case} frame {t} submit_host out_color", want[t], got_piped[t][1])
            if composed:
                _diff(f"{case} frame {t} submit_host out_composed", got_sync[t][0], got_piped[t][0])
        for c in chains:
            c.close()
    finally:
        ctx.close()


def test_statuses(built):
    """is_debug in p; the stage with the tail on and the tail with the stage on; no direct light; out_color with neither stage nor tail;
    both outputs NULL; output 9 with the stage off.  After each refusal the chain still renders."""
    inp = ch.make_inputs(96, 64, 2)
    W, H = inp.width, inp.height
    ctx = _context(inp)
    lib = ctx.lib
    try:
        fr = inp.frames[0]
        fp = [ctx.upload(fr[k]) for k in IN]
        for kw in (dict(), dict(mode=abi.MODE_SSR)):
            c = engine.SsgiChain(ctx, ch.chain_options(inp, ch.Opts(**kw)))
            p = compose_params(fr["cam"], "fog")

            def renders():
                c.render(abi.make_camera(fr["cam"]), *fp, fr["cam"]["position"], True)
                ctx.sync()

            assert lib.rfx_ssgi_chain_output(c.h, 9, C.byref(abi.Plane())) == INVALID_ARG
            bad = compose_params(fr["cam"], "fog")
            bad.is_debug = 1
            assert lib.rfx_ssgi_chain_set_compose(c.h, C.byref(bad)) == INVALID_ARG
            renders()
            c.enable_traa()
            assert lib.rfx_ssgi_chain_set_compose(c.h, C.byref(p)) == INVALID_ARG
            renders()
            c.enable_traa(enable=False)
            assert lib.rfx_ssgi_chain_set_compose(c.h, C.byref(p)) == 0
            assert lib.rfx_ssgi_chain_enable_traa(c.h, C.byref(abi.make_traa_tail_options())) == INVALID_ARG
            renders()
            f = c._frame(abi.make_camera(fr["cam"]), fp[0], fp[1], fp[2], None, fr["cam"]["position"], True)
            assert lib.rfx_ssgi_chain_render(c.h, None, C.byref(f)) == INVALID_ARG
            renders()
            assert lib.rfx_ssgi_chain_output(c.h, 9, C.byref(abi.Plane())) == 0
            hs = {k: np.ascontiguousarray(fr[k]) for k in IN}
            color = np.zeros((H, W, 4), np.float16)
            hf = c.host_frame(abi.make_camera(fr["cam"]), hs["depth"], hs["gbuffer"], hs["velocity"], hs["direct"], fr["cam"]["position"], True)
            assert lib.rfx_ssgi_chain_render_host(c.h, C.byref(hf)) == INVALID_ARG  # both outputs NULL
            hf.out_color = color.ctypes.data
            assert lib.rfx_ssgi_chain_render_host(c.h, C.byref(hf)) == 0
            assert lib.rfx_ssgi_chain_set_compose(c.h, None) == 0
            assert lib.rfx_ssgi_chain_output(c.h, 9, C.byref(abi.Plane())) == INVALID_ARG
            assert lib.rfx_ssgi_chain_render_host(c.h, C.byref(hf)) == NOT_READY  # out_color with neither the stage nor the tail
            renders()
            c.enable_traa()
            assert lib.rfx_ssgi_chain_render_host(c.h, C.byref(hf)) == 0  # the tail's image
            c.close()
        for q in fp:
            q.free()
    finally:
        ctx.close()


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_inprocess_group_with_the_stage_equals_one_chain(built, world):
    """N bands on one GPU, borders moved between frames, the stage off in frame 3: every rank's band of output 9 (and output 0) equals one
    chain's"""
    W, H = 128, 64 * world + 112
    inp = ch.make_inputs(W, H, 5, fov=75.0)
    ctx = _context(inp)
    try:
        copt = ch.chain_options(inp, ch.Opts())
        single, grp = engine.SsgiChain(ctx, copt), parallel.InProcessGroup(ctx, copt, world)
        b = list(grp.bounds)
        for t, fr in enumerate(inp.frames):
            if t in (2, 4):
                grp.set_bounds([0] + [x + (16 if t == 2 else -8) for x in b[1:-1]] + [H])
            p = compose_params(fr["cam"], "exp2") if t != 3 else None
            single.set_compose(p)
            grp.set_compose(p)
            planes = [ctx.upload(fr[k]) for k in IN]
            cam = abi.make_camera(fr["cam"])
            single.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            grp.render(cam, *planes, fr["cam"]["position"], fr["moved"])
            for which in ((0, 9) if p is not None else (0,)):
                _diff(f"world {world} frame {t} output {which} bounds {grp._last_bounds}", single.download(which), grp.download(which))
            for q in planes:
                q.free()
        grp.close()
        single.close()
    finally:
        ctx.close()


def test_sharded_submit_host_downloads_the_band_image(built):
    """a rank-0 group member of a one-rank group: ShardedSsgiChain.submit_host(out_color=...) over pinned host planes gives, frame for frame,
    render_host's image (and `composed`)"""
    inp = ch.make_inputs(160, 128, 4)
    W, H = inp.width, inp.height
    ctx = _context(inp)
    try:
        copt = ch.chain_options(inp, ch.Opts())
        uid = C.create_string_buffer(abi.GROUP_ID_BYTES)
        ctx._chk(ctx.lib.rfx_group_get_unique_id(uid))
        sh = parallel.ShardedSsgiChain(ctx, copt, rank=0, world=1, unique_id=bytes(uid.raw), rebalance_every=0)
        one = engine.SsgiChain(ctx, copt)
        hosts = [{k: _pinned(fr[k]) for k in IN} for fr in inp.frames]
        outs = [(torch.zeros((H, W, 4), dtype=torch.float32).pin_memory(), torch.zeros((H, W, 4), dtype=torch.float16).pin_memory()) for _ in inp.frames]
        with pytest.raises(abi.RfxError, match=f"status {NOT_READY}"):
            sh.submit_host(abi.make_camera(inp.frames[0]["cam"]), hosts[0], inp.frames[0]["cam"]["position"], True, None, outs[0][1])
        bands = []
        for t, fr in enumerate(inp.frames):
            p = compose_params(fr["cam"], "fog")
            sh.set_compose(p)
            bands.append(sh.submit_host(abi.make_camera(fr["cam"]), hosts[t], fr["cam"]["position"], fr["moved"], outs[t][0], out_color=outs[t][1]))
            sh.wait_host(1)
        sh.wait_host(0)
        for t, fr in enumerate(inp.frames):
            one.set_compose(compose_params(fr["cam"], "fog"))
            want_c, want_i = np.zeros((H, W, 4), np.float32), np.zeros((H, W, 4), np.float16)
            one.render_host(one.host_frame(abi.make_camera(fr["cam"]), *(hosts[t][k] for k in IN), fr["cam"]["position"], fr["moved"], want_c, want_i))
            assert bands[t] == (0, H)
            _diff(f"frame {t} image", want_i, outs[t][1].numpy())
            _diff(f"frame {t} composed", want_c, outs[t][0].numpy())
        one.close()
        sh.close()
    finally:
        ctx.close()
