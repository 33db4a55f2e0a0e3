"""The motion-blur stage of the TRAA tail (rfx_*_chain_set_motion_blur: TRAAEffect + MotionBlurEffect as one EffectPass) at 3840 x 2160 on
one GPU.  Prints one JSON line with the card's name and power limit.

    python tools/bench_mb_tail.py [--frames 100] [--warmup 10] [--width 3840 --height 2160]

Two workloads, each as two chains timed with CUDA events on the context's stream in alternating blocks:
  ssgi_c3   the SSGI + TRAA frame of tools/bench_traa.py (fast chain, denoiseIterations 2): the tail (K5 -> K2 -> K9) against the tail
            with the stage (K5 -> K2 -> the merged TRAA + motion-blur launch);
  ao_c4     the AO frame of tools/bench_ao_traa.py (K6 spp 8, iterations 1, K7): the tail (K2 -> K9) against the tail with the stage, and
            in-process groups of N = 2, 4, 8 bands with the stage (two phases per frame; the members render one after the other on one card,
            so a group's frame is the sum of its members' kernel times and its ratio to the chain with the stage is the cost of sharding).
MotionBlurEffect's defaults (intensity 1, jitter 1, samples 16) at deltaTime 1/60, on the harness's moving camera.  Before the timed region
each chain with the stage is checked byte for byte: its TRAA accumulated plane against the chain without the stage (the TRAA bytes do not
change), and its output against rfx_traa_motion_blur_launch on its own planes; every group's output and TRAA history against the chain with the
stage."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import chain_harness as ch  # noqa: E402
from bench_ao import device_info  # noqa: E402
from realism_effects_b200 import abi, engine, parallel  # noqa: E402

WORLDS = (2, 4, 8)


def _time(a, ctx, step, setups) -> dict:
    import torch

    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    blocks, ms = 4, {s: 0.0 for s in setups}
    for _ in range(blocks):  # alternate the setups so that clock and neighbour load drift hit both alike
        for s in setups:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.frames // blocks):
                step(s)
            e1.record(stream)
            e1.synchronize()
            ms[s] += e0.elapsed_time(e1)
    return {s: ms[s] / (blocks * (a.frames // blocks)) for s in setups}


def ssgi_c3(a) -> dict:
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda", reference_env=True)
    ctx = engine.Context(0, inp.blue)
    ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    copt, topt = ch.chain_options(inp, ch.Opts(denoise_iterations=2)), abi.make_traa_tail_options()
    chains = {s: engine.SsgiChain(ctx, copt) for s in ("tail", "stage")}
    for c in chains.values():
        c.enable_traa(topt)
    p = ch.motion_blur_params(W, H)
    frames = [([ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")], abi.make_camera(fr["cam"]), fr) for fr in inp.frames]
    n = {s: 0 for s in chains}

    def step(s):
        planes, cam, fr = frames[n[s] % len(frames)]
        if s == "stage":
            p.frame = n[s] % 4096
            chains[s].set_motion_blur(p)
        chains[s].render(cam, *planes, fr["cam"]["position"], n[s] > 0)
        n[s] += 1

    for _ in range(a.warmup):
        for s in chains:
            step(s)
    ctx.sync()
    k5, out = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
    planes = frames[(n["stage"] - 1) % len(frames)][0]
    ctx.ssgi_compose(planes[0], chains["stage"].output(0), planes[3], k5, params=topt.compose)
    ctx.traa_motion_blur(p, planes[2], chains["stage"].output(7), k5, out)
    check = {"traa_accumulated_unchanged": chains["stage"].download(7).tobytes() == chains["tail"].download(7).tobytes(),
             "output_equals_per_pass_launch": chains["stage"].download(6).tobytes() == out.download().tobytes()}
    per = _time(a, ctx, step, list(chains))
    for c in chains.values():
        c.close()
    ctx.close()
    return {"workload": f"SSGI C3 at {W}x{H}, denoiseIterations 2, TRAA tail; motion blur samples 16", "frames": a.frames, "warmup": a.warmup,
            "self_check_bit_exact": check, "ms_chain_with_tail": round(per["tail"], 4), "ms_chain_with_tail_and_stage": round(per["stage"], 4),
            "ms_stage": round(per["stage"] - per["tail"], 4)}


def ao_c4(a) -> dict:
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda")
    ctx = engine.Context(0, inp.blue)
    copt, topt = engine.ao_chain_options(W, H, {"iterations": 1}), abi.make_traa_tail_options()
    chains = {s: engine.AoChain(ctx, copt) for s in ("tail", "stage")}
    for c in chains.values():
        c.enable_traa(topt)
    p = ch.motion_blur_params(W, H)
    frames = [(ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"]), fr["cam"]) for fr in inp.frames]
    groups = {w: parallel.InProcessAoGroup(ctx, copt, w, traa=topt, motion_blur=p) for w in WORLDS}
    setups = [*chains, *groups]
    outs = {s: ctx.alloc(abi.FMT_RGBA16F, W, H) for s in setups}
    n = {s: 0 for s in setups}

    def step(s):
        d, v, i, u = frames[n[s] % len(frames)]
        p.frame = n[s] % 4096
        if s in groups:  # no per-frame host wait: one stream orders the members, their phases and the frames
            groups[s].set_motion_blur(p)
            groups[s].render(u, d, v, None, i, outs[s], wait=False, traa_cam=u, camera_moved=True)
        else:
            if s == "stage":
                chains[s].set_motion_blur(p)
            chains[s].render(u, d, v, None, i, outs[s], traa_cam=u, camera_moved=True)
        n[s] += 1

    for _ in range(a.warmup):
        for s in setups:
            step(s)
    ctx.sync()
    out = ctx.alloc(abi.FMT_RGBA16F, W, H)
    vel = frames[(n["stage"] - 1) % len(frames)][1]
    ctx.traa_motion_blur(p, vel, chains["stage"].output(3), chains["stage"].output(2), out)
    check = {"traa_accumulated_unchanged": chains["stage"].download(3).tobytes() == chains["tail"].download(3).tobytes(),
             "output_equals_per_pass_launch": outs["stage"].download().tobytes() == out.download().tobytes()}
    for w, g in groups.items():
        check[f"group_n{w}"] = (outs[w].download().tobytes() == outs["stage"].download().tobytes()
                                and g.download(3).tobytes() == chains["stage"].download(3).tobytes())
    per = _time(a, ctx, step, setups)
    for g in groups.values():
        g.close()
    for c in chains.values():
        c.close()
    ctx.close()
    return {"workload": f"AO C4 (K6 spp 8) at {W}x{H}, iterations 1, K7, TRAA tail; motion blur samples 16", "frames": a.frames, "warmup": a.warmup,
            "self_check_bit_exact": check, "ms_chain_with_tail": round(per["tail"], 4), "ms_chain_with_tail_and_stage": round(per["stage"], 4),
            "ms_stage": round(per["stage"] - per["tail"], 4),
            **{f"ms_group_n{w}_sum_of_members": round(per[w], 4) for w in WORLDS},
            **{f"overhead_n{w}": round(per[w] / per["stage"], 4) for w in WORLDS}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_mb_tail.py measures on the GPU; there is no CPU timing"
    assert a.frames >= 100 and a.warmup >= 2, "at least 100 timed frames and 2 warm-up frames"
    res = {"device": device_info(0), "ssgi_c3": ssgi_c3(a), "ao_c4": ao_c4(a)}
    res["self_check_passed"] = all(all(res[k]["self_check_bit_exact"].values()) for k in ("ssgi_c3", "ao_c4"))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
