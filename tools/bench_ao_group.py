"""The native AO chain and its row-sharded groups: C4 (HBAOEffect's defaults: K6 with spp 8) and C4-literal (K6h, 8 directions x 32
steps), each with iterations 1 (one Poisson pass pair) and K7, at 3840 x 2160.  Prints one JSON line.

    python tools/bench_ao_group.py [--frames 100] [--warmup 10] [--width 3840 --height 2160]
    python -m torch.distributed.run --nproc_per_node N tools/bench_ao_group.py     # + ms per frame per rank, and 7680 x 4320

One GPU: the per-pass effect class (HBAOEffect / HorizonAOEffect: one launch call per pass from Python), one AoChain (the same launches
in one call), and in-process groups of N = 2, 4, 8 bands (one context: the members render one after the other on one stream, so a group's
frame is the sum of its members' kernel times; its ratio to the plain chain is the cost of row-sharding on one card, the halo rows every
member recomputes).  Setups are timed with CUDA events in alternating blocks.  Before the timed region every setup's denoised plane and
composed output are compared with the plain chain's byte for byte (self_check)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import chain_harness as ch  # noqa: E402
from bench_ao import device_info  # noqa: E402
from realism_effects_b200 import abi, effects, engine, parallel  # noqa: E402

WORKLOADS = {"c4_spp8": (False, {"iterations": 1}), "c4_literal_horizon_8x32": (True, {"iterations": 1, "directions": 8, "steps": 32})}
WORLDS = (2, 4, 8)


class _Scene:
    def __init__(self, depth, velocity):
        self.depth, self.velocity = depth, velocity


class _Composer:
    def __init__(self, ctx, w, h, inp):
        self.ctx, self.width, self.height, self.inputBuffer = ctx, w, h, inp
        self.outputBuffer = ctx.alloc(abi.FMT_RGBA16F, w, h)


class _Cam:
    u = None

    def uniforms(self):
        return self.u


def one_gpu(a, name) -> dict:
    import torch

    horizon, opts = WORKLOADS[name]
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda")
    ctx = engine.Context(0, inp.blue)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    frames = [(ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"]), fr["cam"]) for fr in inp.frames]
    copt = engine.ao_chain_options(W, H, opts, horizon=horizon)
    plain = engine.AoChain(ctx, copt)
    groups = {n: parallel.InProcessAoGroup(ctx, copt, n) for n in WORLDS}
    outs = {s: ctx.alloc(abi.FMT_RGBA16F, W, H) for s in ("plain", *WORLDS)}
    cam, scene = _Cam(), _Scene(*frames[0][:2])
    comp = _Composer(ctx, W, H, frames[0][2])
    fx = (effects.HorizonAOEffect if horizon else effects.HBAOEffect)(comp, cam, scene, opts)
    count = {s: 0 for s in ("effect", "plain", *WORLDS)}

    def step(s):
        d, v, i, u = frames[count[s] % len(frames)]
        if s == "effect":
            cam.u, scene.depth, scene.velocity, comp.inputBuffer = u, d, v, i
            fx.update(None, i)
        elif s == "plain":
            plain.render(u, d, v, None, i, outs[s])
        else:  # no per-frame host wait: one stream orders the members and the frames
            groups[s].render(u, d, v, None, i, outs[s], wait=False)
        count[s] += 1

    check = {}
    for i in range(a.warmup):
        for s in count:
            step(s)
        if i in (0, a.warmup - 1):  # bit-exact against the plain chain before the timed region
            ctx.sync()
            ref = (plain.download(1).tobytes(), outs["plain"].download().tobytes())
            got = {"effect": (fx.texture.download().tobytes(), comp.outputBuffer.download().tobytes())}
            for n in WORLDS:
                got[f"n{n}"] = (groups[n].download(1).tobytes(), outs[n].download().tobytes())
            for k, v in got.items():
                check[k] = check.get(k, True) and v == ref
    ctx.sync()
    blocks = 4
    ms = {s: 0.0 for s in count}
    for _ in range(blocks):  # alternate the setups so that clock and neighbour load drift hit all of them alike
        for s in count:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.frames // blocks):
                step(s)
            e1.record(stream)
            e1.synchronize()
            ms[s] += e0.elapsed_time(e1)
    nf = blocks * (a.frames // blocks)
    per = {s: ms[s] / nf for s in ms}
    res = {"workload": f"{name} at {W}x{H}, iterations 1, K7; per-pass effect vs AoChain vs in-process groups on one GPU", "frames": nf,
           "warmup": a.warmup, "self_check_bit_exact": check, "ms_effect_per_pass": round(per["effect"], 4), "ms_chain": round(per["plain"], 4)}
    for n in WORLDS:
        res[f"ms_group_n{n}_sum_of_members"] = round(per[n], 4)
        res[f"overhead_n{n}"] = round(per[n] / per["plain"], 4)
    for g in groups.values():
        g.close()
    plain.close()
    fx.dispose()
    ctx.close()
    return res


def multi_gpu(a, rank, world, name, W, H) -> dict:
    """W x H row-sharded over `world` GPUs (one process each): ms per frame of every rank"""
    import torch
    import torch.distributed as dist

    horizon, opts = WORKLOADS[name]
    torch.cuda.set_device(rank)
    inp = ch.make_inputs(W, H, 2, device="cuda")
    ctx = engine.Context(rank, inp.blue)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", rank))
    sh = parallel.ShardedAoChain(ctx, engine.ao_chain_options(W, H, opts, horizon=horizon))
    frames = [(ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"]), fr["cam"]) for fr in inp.frames]
    out = ctx.alloc(abi.FMT_RGBA16F, W, H)
    for i in range(a.warmup):
        d, v, x, u = frames[i % 2]
        sh.render(u, d, v, None, x, out)
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(a.frames):
        d, v, x, u = frames[i % 2]
        sh.render(u, d, v, None, x, out)
    e1.record(stream)
    e1.synchronize()
    t = torch.zeros(world, device=f"cuda:{rank}")
    t[rank] = e0.elapsed_time(e1) / a.frames
    dist.all_reduce(t)
    sh.close()
    ctx.close()
    return {"workload": f"{name} at {W}x{H} row-sharded over {world} GPUs", "frames": a.frames, "ms_per_frame_per_rank": [round(float(x), 4) for x in t.tolist()]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_ao_group.py measures on the GPU; there is no CPU timing"
    assert a.frames >= 100 and a.warmup >= 2, "at least 100 timed frames and 2 warm-up frames"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    res = {"device": device_info(rank)}
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("gloo")
        for name in WORKLOADS:
            res[f"{name}_sharded"] = multi_gpu(a, rank, world, name, a.width, a.height)
            res[f"{name}_8k"] = multi_gpu(a, rank, world, name, 7680, 4320)
        dist.destroy_process_group()
    if rank == 0:
        for name in WORKLOADS:
            res[name] = one_gpu(a, name)
        res["self_check_passed"] = all(all(res[n]["self_check_bit_exact"].values()) for n in WORKLOADS)
        print(json.dumps(res))


if __name__ == "__main__":
    main()
