"""The AO chain's TRAA frame tail (rfx_ao_chain_enable_traa): C4 (HBAOEffect's defaults: K6 with spp 8) and C4-literal (K6h, 8 directions x
32 steps), each with iterations 1 and K7, at 3840 x 2160.  Prints one JSON line.

    python tools/bench_ao_traa.py [--frames 100] [--warmup 10] [--width 3840 --height 2160]

One GPU, one context, one stream: the AO chain alone (K6 -> Poisson x 2 -> K7), the chain with the tail (+ TRAA's K2 and K9), the per-pass
effects (HBAOEffect / HorizonAOEffect, then TRAAEffect.update and compose: one launch call per pass from Python), and in-process groups of
N = 2, 4, 8 bands with the tail (the members render one after the other, so a group's frame is the sum of its members' kernel times; its
ratio to the chain with the tail is the cost of row-sharding on one card).  Setups are timed with CUDA events in alternating blocks.  Before
the timed region the K9 output and the TRAA accumulated plane of every setup with the tail are compared with the chain's byte for byte
(self_check)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import chain_harness as ch  # noqa: E402
from bench_ao import device_info  # noqa: E402
from bench_ao_group import WORKLOADS, WORLDS, _Cam, _Composer, _Scene  # noqa: E402
from realism_effects_b200 import abi, effects, engine, parallel  # noqa: E402


class _VelocityPass:
    texture = None


def one_gpu(a, name) -> dict:
    import torch

    horizon, opts = WORKLOADS[name]
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda")
    ctx = engine.Context(0, inp.blue)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    frames = [(ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"]), fr["cam"]) for fr in inp.frames]
    copt = engine.ao_chain_options(W, H, opts, horizon=horizon)
    topt = abi.make_traa_tail_options()
    plain, tail = engine.AoChain(ctx, copt), engine.AoChain(ctx, copt)
    tail.enable_traa(topt)
    groups = {n: parallel.InProcessAoGroup(ctx, copt, n, traa=topt) for n in WORLDS}
    outs = {s: ctx.alloc(abi.FMT_RGBA16F, W, H) for s in ("plain", "tail", "effects", *WORLDS)}
    cam, scene, vel = _Cam(), _Scene(*frames[0][:2]), _VelocityPass()
    comp = _Composer(ctx, W, H, frames[0][2])
    fx = (effects.HorizonAOEffect if horizon else effects.HBAOEffect)(comp, cam, scene, opts)
    traa = effects.TRAAEffect(None, cam, vel)
    # the chain's tail starts with keepData 0: a TemporalReprojectPass reset before its first frame
    traa.temporalReprojectPass = effects.TemporalReprojectPass(None, cam, vel, comp.outputBuffer, 1, traa.options)
    traa.reset()
    count = {s: 0 for s in ("plain", "tail", "effects", *WORLDS)}

    def step(s):
        d, v, i, u = frames[count[s] % len(frames)]  # the two frames alternate: the camera moves on every frame
        if s == "effects":
            cam.u, scene.depth, scene.velocity, comp.inputBuffer, vel.texture = u, d, v, i, v
            fx.update(None, i)
            traa.update(None, comp.outputBuffer)
            traa.compose(outs[s])
        elif s == "plain":
            plain.render(u, d, v, None, i, outs[s])
        elif s == "tail":
            tail.render(u, d, v, None, i, outs[s], traa_cam=u, camera_moved=True)
        else:  # no per-frame host wait: one stream orders the members and the frames
            groups[s].render(u, d, v, None, i, outs[s], wait=False, traa_cam=u, camera_moved=True)
        count[s] += 1

    check = {}
    for i in range(a.warmup):
        for s in count:
            step(s)
        if i in (0, a.warmup - 1):  # bit-exact against the chain with the tail before the timed region
            ctx.sync()
            ref = (tail.download(3).tobytes(), outs["tail"].download().tobytes())
            got = {"effects": (traa.temporalReprojectPass.accumulated.download().tobytes(), outs["effects"].download().tobytes())}
            for n in WORLDS:
                got[f"n{n}"] = (groups[n].download(3).tobytes(), outs[n].download().tobytes())
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
    res = {"workload": f"{name} at {W}x{H}, iterations 1, K7, TRAA tail; AoChain alone / with the tail / per-pass effects / in-process groups",
           "frames": nf, "warmup": a.warmup, "self_check_bit_exact": check, "ms_chain": round(per["plain"], 4), "ms_chain_with_tail": round(per["tail"], 4),
           "ms_tail": round(per["tail"] - per["plain"], 4), "ms_effects_per_pass": round(per["effects"], 4)}
    for n in WORLDS:
        res[f"ms_group_n{n}_sum_of_members"] = round(per[n], 4)
        res[f"overhead_n{n}"] = round(per[n] / per["tail"], 4)
    for g in groups.values():
        g.close()
    plain.close()
    tail.close()
    fx.dispose()
    traa.dispose()
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_ao_traa.py measures on the GPU; there is no CPU timing"
    assert a.frames >= 100 and a.warmup >= 2, "at least 100 timed frames and 2 warm-up frames"
    res = {"device": device_info(0)}
    for name in WORKLOADS:
        res[name] = one_gpu(a, name)
    res["self_check_passed"] = all(all(res[n]["self_check_bit_exact"].values()) for n in WORKLOADS)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
