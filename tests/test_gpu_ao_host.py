"""The AO chain's host-buffer path on the GPU (rfx_ao_chain_render_host / _submit_host / _wait_host, parallel.ShardedAoChain.submit_host):
frames from host memory give the bytes of the same chain rendering device planes, frame after frame, synchronously and pipelined; every
refusal returns its status and a message; a row-sharded group of one rank, and of two processes with moving borders, gives each rank's
band of the one-GPU frame."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

import ao_harness as ao
import chain_harness as ch
from realism_effects_b200 import abi, effects, engine, parallel
from test_gpu_ao_chain import HORIZON_SMALL, _diff

pytestmark = pytest.mark.gpu

W, H = 96, 160  # two bands of >= 64 rows (what a row-sharded group takes)
STAGES = ["k7", "no-k7", "tail", "tail+blur"]  # K7 into out_color; no input (out_ao only); the TRAA tail; the tail with the motion-blur stage


def _blur(t: int) -> abi.MotionBlurParams:
    p = ch.motion_blur_params(W, H, frame=t, samples=16, delta_time=1 / 1000 if t % 2 == 0 else 1 / 60)
    p.intensity = 3.0
    return p


class Frames:
    """5 moving frames (a camera that pans, a rotating velocity field that changes every frame) as host arrays, and didCameraMove"""

    def __init__(self, use_normal: bool, n: int = 5):
        inp = ch.make_inputs(W, H, n)
        self.blue = inp.blue
        self.frames, prev = [], None
        for t, fr in enumerate(inp.frames):
            vel = np.array(fr["velocity"], copy=True)
            vel[..., :2] = ch.rotation_velocity_field(W, H, fr["depth"], 0.01 + 0.005 * t)[..., :2]
            self.frames.append(dict(cam=fr["cam"], depth=np.ascontiguousarray(fr["depth"]), velocity=vel, input=np.ascontiguousarray(fr["direct"]),
                                    normal=np.ascontiguousarray(ao.view_normal_plane(W, H, t, fr["cam"])) if use_normal else None,
                                    moved=effects._did_camera_move(fr["cam"], prev)))
            prev = fr["cam"]


def _chain(ctx, horizon, iterations, use_normal, scale, stage):
    opts = {"blueNoiseStart": 777, "iterations": iterations, "useNormalPass": use_normal, "resolutionScale": scale, **(HORIZON_SMALL if horizon else {})}
    c = engine.AoChain(ctx, engine.ao_chain_options(W, H, opts, horizon=horizon))
    if stage.startswith("tail"):
        c.enable_traa(abi.make_traa_tail_options(full_accumulate=True))
    if stage == "tail+blur":
        c.set_motion_blur(_blur(0))
    return c


def _device_frame(ctx, chain, fr, t, stage, out):
    """the reference: the chain on device planes (rfx_ao_chain_render / _render_traa); returns out_color, out_ao and outputs 0..3"""
    planes = [ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["normal"]) if fr["normal"] is not None else None,
              ctx.upload(fr["input"]) if stage != "no-k7" else None]
    if stage == "tail+blur":
        chain.set_motion_blur(_blur(t))
    tail = stage.startswith("tail")
    chain.render(fr["cam"], *planes, out if stage != "no-k7" else None, traa_cam=fr["cam"] if tail else None, camera_moved=fr["moved"])
    got = _outputs(chain, tail, out.download() if stage != "no-k7" else None, chain.download(1))
    for p in planes:
        if p is not None:
            p.free()
    return got


def _outputs(chain, tail, color, ao_plane):
    return dict(color=color, ao=ao_plane, **{f"output {w}": chain.download(w) for w in ((0, 1, 2, 3) if tail else (0, 1))})


class HostSet:
    """one set of host buffers of a frame (pinned: the pipelined copies are asynchronous)"""

    def __init__(self, ao_shape):
        z = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory()  # noqa: E731
        self.depth, self.velocity = z((H, W), torch.float32), z((H, W, 4), torch.float32)
        self.normal, self.input = z((H, W, 4), torch.uint8), z((H, W, 4), torch.float16)
        self.color, self.ao = z((H, W, 4), torch.float16), z(ao_shape, torch.float16)

    def fill(self, fr):
        for k in ("depth", "velocity", "normal", "input"):
            if fr.get(k) is not None:
                getattr(self, k).copy_(torch.from_numpy(np.ascontiguousarray(fr[k])))

    def scribble(self):
        for t in (self.depth, self.velocity, self.normal, self.input, self.color, self.ao):
            t.view(torch.uint8).fill_(0x5a)

    def frame(self, chain, fr, stage):
        k7 = stage != "no-k7"
        return chain.host_frame(fr["cam"], self.depth, self.velocity, self.normal if fr["normal"] is not None else None, self.input if k7 else None,
                                self.color if k7 else None, self.ao, traa_cam=fr["cam"] if stage.startswith("tail") else None, camera_moved=fr["moved"])


def _ao_shape(chain):
    p = chain.output(1)
    return (p.height, p.width, 4)


@pytest.mark.parametrize("stage", STAGES)
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("use_normal", [False, True], ids=["depth-normal", "normal-plane"])
@pytest.mark.parametrize("iterations", [0, 2])
@pytest.mark.parametrize("horizon", [False, True], ids=["hbao", "horizon"])
def test_render_host_equals_render(built, horizon, iterations, use_normal, scale, stage):
    """Over 5 moving frames render_host (numpy host arrays) writes the bytes of render on device planes into out_color and out_ao, and
    leaves outputs 0..3 equal to the device-path chain's"""
    fs = Frames(use_normal)
    ctx = engine.Context(0, fs.blue)
    try:
        dev, host = (_chain(ctx, horizon, iterations, use_normal, scale, stage) for _ in range(2))
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        for t, fr in enumerate(fs.frames):
            want = _device_frame(ctx, dev, fr, t, stage, out)
            color, ao_plane = np.full((H, W, 4), np.nan, np.float16), np.full(_ao_shape(host), np.nan, np.float16)
            if stage == "tail+blur":
                host.set_motion_blur(_blur(t))
            k7 = stage != "no-k7"
            hf = host.host_frame(fr["cam"], fr["depth"], fr["velocity"], fr["normal"], fr["input"] if k7 else None, color if k7 else None, ao_plane,
                                 traa_cam=fr["cam"] if stage.startswith("tail") else None, camera_moved=fr["moved"])
            host.render_host(hf)
            got = _outputs(host, stage.startswith("tail"), color if k7 else None, ao_plane)
            for k, v in want.items():
                if v is not None:
                    _diff(f"frame {t} {k}", v, got[k])
        for c in (dev, host):
            c.close()
        out.free()
    finally:
        ctx.close()


@pytest.mark.parametrize("case", [dict(horizon=False, iterations=2, use_normal=False, stage="tail+blur"),
                                  dict(horizon=True, iterations=0, use_normal=True, stage="k7"),
                                  dict(horizon=False, iterations=1, use_normal=True, stage="no-k7"),
                                  dict(horizon=True, iterations=2, use_normal=False, stage="tail")], ids=lambda c: f"{c['stage']}-it{c['iterations']}")
def test_pipelined_submit_host_equals_render(built, case):
    """submit_host / wait_host(1) over two host buffer sets: after each wait the released set's buffers (inputs and downloads) are
    overwritten at once, so an upload or download that ran late would show up.  Every frame equals the device path."""
    fs = Frames(case["use_normal"], n=6)
    stage = case["stage"]
    ctx = engine.Context(0, fs.blue)
    try:
        dev, host = (_chain(ctx, case["horizon"], case["iterations"], case["use_normal"], 1.0, stage) for _ in range(2))
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        want = [_device_frame(ctx, dev, fr, t, stage, out) for t, fr in enumerate(fs.frames)]
        sets = [HostSet(_ao_shape(host)) for _ in range(2)]
        got, hfs = [], [None, None]

        def collect(i):
            s = sets[i % 2]
            got.append(dict(color=s.color.numpy().copy() if stage != "no-k7" else None, ao=s.ao.numpy().copy()))
            s.scribble()  # the set is released: the next frame that uses it must not see any of this frame's bytes, nor this frame these

        for i, fr in enumerate(fs.frames):
            s = sets[i % 2]
            s.fill(fr)
            hfs[i % 2] = s.frame(host, fr, stage)
            if stage == "tail+blur":
                host.set_motion_blur(_blur(i))
            host.submit_host(hfs[i % 2])
            host.wait_host(1)
            if i >= 1:
                collect(i - 1)
        host.wait_host(0)
        collect(len(fs.frames) - 1)
        for t, (w, g) in enumerate(zip(want, got)):
            for k in ("color", "ao"):
                if w[k] is not None:
                    _diff(f"frame {t} {k}", w[k], g[k])
        for k, v in _outputs(dev, stage.startswith("tail"), None, None).items():  # the chains' own planes after the last frame
            if v is not None:
                _diff(f"last frame {k}", v, _outputs(host, stage.startswith("tail"), None, None)[k])
        for c in (dev, host):
            c.close()
        out.free()
    finally:
        ctx.close()


def _status(lib, ctx, st, want):
    msg = lib.rfx_last_error(ctx.h).decode()
    assert st == want and msg, (st, want, msg)
    return msg


def test_statuses(built):
    """1 = RFX_ERR_INVALID_ARG, 5 = RFX_ERR_NOT_READY, 6 = RFX_ERR_UNSUPPORTED (include/rfx.h); a refused call leaves the chain usable"""
    fs = Frames(True, n=2)
    fr = fs.frames[0]
    ctx = engine.Context(0, fs.blue)
    lib = ctx.lib
    try:
        copt = engine.ao_chain_options(W, H, {"iterations": 1, "useNormalPass": True})
        chain = engine.AoChain(ctx, copt)
        color, ao_plane = np.zeros((H, W, 4), np.float16), np.zeros((H, W, 4), np.float16)
        full = dict(depth=fr["depth"], velocity=fr["velocity"], normal=fr["normal"], inp=fr["input"], out_color=color, out_ao=ao_plane)

        def submit(**kw):
            return lib.rfx_ao_chain_submit_host(chain.h, C.byref(chain.host_frame(fr["cam"], **{**full, **kw})))

        for kw in (dict(depth=None), dict(velocity=None), dict(normal=None), dict(out_color=None), dict(inp=None, out_color=None, out_ao=None),
                   dict(inp=None)):
            _status(lib, ctx, submit(**kw), 1)
        assert lib.rfx_ao_chain_render_host(chain.h, C.byref(chain.host_frame(fr["cam"], **{**full, "depth": None}))) == 1
        for n in (-1, 2):
            _status(lib, ctx, lib.rfx_ao_chain_wait_host(chain.h, n), 1)
        # a TRAA camera with the tail off is not ready; with the tail on, the camera and the colour planes are required
        _status(lib, ctx, lib.rfx_ao_chain_submit_host(chain.h, C.byref(chain.host_frame(fr["cam"], **full, traa_cam=fr["cam"]))), 5)
        chain.enable_traa()
        _status(lib, ctx, submit(), 1)
        _status(lib, ctx, lib.rfx_ao_chain_submit_host(chain.h, C.byref(chain.host_frame(fr["cam"], **{**full, "inp": None, "out_color": None},
                                                                                             traa_cam=fr["cam"]))), 1)
        chain.enable_traa(enable=False)
        chain.render_host(chain.host_frame(fr["cam"], **full))  # still usable
        chain.close()
        # a member of a group of n > 1: unsupported; between the two phases of a frame with the motion-blur stage: not ready
        d, v, n, i = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["normal"]), ctx.upload(fr["input"])
        out = ctx.alloc(abi.FMT_RGBA16F, W, H)
        grp = parallel.InProcessAoGroup(ctx, copt, 2)
        m = grp.chains[0]
        _status(lib, ctx, lib.rfx_ao_chain_submit_host(m.h, C.byref(m.host_frame(fr["cam"], **full))), 6)
        grp.close()
        grp = parallel.InProcessAoGroup(ctx, copt, 2, traa=abi.make_traa_tail_options(), motion_blur=_blur(0))
        tf = grp.chains[0]._traa_frame(fr["cam"], True)
        for m in grp.chains:
            assert lib.rfx_ao_chain_render_sharded_traa(m.h, None, C.byref(m._frame(fr["cam"], d, v, n, i, out)), C.byref(tf)) == 0
        m = grp.chains[0]
        msg = _status(lib, ctx, lib.rfx_ao_chain_submit_host(m.h, C.byref(m.host_frame(fr["cam"], **full, traa_cam=fr["cam"]))), 5)
        assert "render_sharded_finish" in msg
        grp._finish(True)
        grp.close()
        for p in (d, v, n, i, out):
            p.free()
    finally:
        ctx.close()


def _host_tensors(fr, stage):
    keys = ("depth", "velocity", "normal") + (("input",) if stage != "no-k7" else ())
    return {k: torch.from_numpy(np.ascontiguousarray(fr[k])).pin_memory() for k in keys if fr.get(k) is not None}


def _sharded_frames(sh, fs, stage):
    """every frame through ShardedAoChain.submit_host / wait_host(1): [(band, rows of the download)]"""
    outs = [torch.zeros((H, W, 4), dtype=torch.float16).pin_memory() for _ in fs.frames]
    hosts = [_host_tensors(fr, stage) for fr in fs.frames]
    bands = []
    for j, fr in enumerate(fs.frames):
        bands.append(sh.submit_host(fr["cam"], hosts[j], outs[j]))
        sh.wait_host(1)
    sh.wait_host(0)
    return [((b0, b1), o.numpy()[: b1 - b0].copy()) for o, (b0, b1) in zip(outs, bands)]


def _one_gpu_downloads(ctx, fs, opts, stage):
    """render_host on one chain: the frame's out_color (with K7) or out_ao"""
    chain = engine.AoChain(ctx, engine.ao_chain_options(W, H, opts))
    res = []
    for fr in fs.frames:
        color, ao_plane = np.zeros((H, W, 4), np.float16), np.zeros((H, W, 4), np.float16)
        k7 = stage != "no-k7"
        chain.render_host(chain.host_frame(fr["cam"], fr["depth"], fr["velocity"], fr["normal"], fr["input"] if k7 else None,
                                           color if k7 else None, ao_plane))
        res.append(color if k7 else ao_plane)
    chain.close()
    return res


@pytest.mark.parametrize("stage", ["k7", "no-k7"])
def test_sharded_host_path_of_one_rank_equals_render_host(built, stage):
    fs = Frames(True)
    opts = {"iterations": 2, "useNormalPass": True}
    ctx = engine.Context(0, fs.blue)
    try:
        want = _one_gpu_downloads(ctx, fs, opts, stage)
        uid = C.create_string_buffer(abi.GROUP_ID_BYTES)
        ctx._chk(ctx.lib.rfx_group_get_unique_id(uid))
        sh = parallel.ShardedAoChain(ctx, engine.ao_chain_options(W, H, opts), rank=0, world=1, unique_id=bytes(uid.raw))
        for t, ((b0, b1), rows) in enumerate(_sharded_frames(sh, fs, stage)):
            assert (b0, b1) == (0, H)
            _diff(f"frame {t}", want[t], rows)
        h2d, d2h = sh.host_bytes_per_frame
        assert d2h == H * W * 8 and h2d == H * W * (4 + 16 + 4 + (8 if stage == "k7" else 0))
        sh.close()
        ctx._chk(ctx.lib.rfx_group_get_unique_id(uid))  # a new group: a new id
        with pytest.raises(abi.RfxError, match="status 6"):
            sh2 = parallel.ShardedAoChain(ctx, engine.ao_chain_options(W, H, opts), rank=0, world=1, unique_id=bytes(uid.raw),
                                          traa=abi.make_traa_tail_options())
            try:
                sh2.submit_host(fs.frames[0]["cam"], _host_tensors(fs.frames[0], "k7"), torch.zeros((H, W, 4), dtype=torch.float16))
            finally:
                sh2.close()
    finally:
        ctx.close()


# ---- two processes, one GPU each -------------------------------------------------------------------------------------------------------------
def _worker(rank, world, port, q, case):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fs = Frames(case["use_normal"])
        ctx = engine.Context(rank, fs.blue)
        sh = parallel.ShardedAoChain(ctx, engine.ao_chain_options(W, H, case["opts"]), rebalance_every=0)
        bands = [[0, H // 2 - 16 + 8 * j, H] for j in range(len(fs.frames))]  # borders that move every frame
        rows = []
        outs = [torch.zeros((H, W, 4), dtype=torch.float16).pin_memory() for _ in fs.frames]
        hosts = [_host_tensors(fr, case["stage"]) for fr in fs.frames]
        for j, fr in enumerate(fs.frames):
            sh.set_bounds(bands[j])
            rows.append(sh.submit_host(fr["cam"], hosts[j], outs[j]))
            sh.wait_host(1)
        sh.wait_host(0)
        q.put((rank, [((b0, b1), o.numpy()[: b1 - b0].tobytes()) for o, (b0, b1) in zip(outs, rows)]))
        sh.close()
        ctx.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("case", [dict(opts={"iterations": 1}, use_normal=False, stage="k7"),
                                  dict(opts={"iterations": 2, "useNormalPass": True}, use_normal=True, stage="no-k7")], ids=["k7", "no-k7"])
def test_two_gpu_sharded_host_path_equals_one_gpu(built, case):
    """Two processes, borders moved every frame: each rank's band of the download equals one GPU's render_host rows"""
    import torch.multiprocessing as mp

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
    fs = Frames(case["use_normal"])
    ctx = engine.Context(0, fs.blue)
    try:
        want = _one_gpu_downloads(ctx, fs, case["opts"], case["stage"])
    finally:
        ctx.close()
    borders = set()
    for rank in range(2):
        for t, ((b0, b1), got) in enumerate(res[rank]):
            borders.add((rank, b0, b1))
            assert got == want[t][b0:b1].tobytes(), (rank, t, (b0, b1))
    assert len(borders) > 2  # the borders moved
