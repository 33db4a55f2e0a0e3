"""Row-sharded groups of the per-pass chain: SSR with the reference demo's options (denoiseMode "full_temporal", everything else default) and
SSGI in denoiseMode "full_temporal", at 3840 x 2160 with the demo HDR environment.  Prints one JSON line.

    python tools/bench_group_modes.py [--frames 100] [--warmup 10] [--width 3840 --height 2160]
    python -m torch.distributed.run --nproc_per_node N tools/bench_group_modes.py     # + ms per frame per rank and C5 (7680 x 4320)

One GPU: in-process groups of N = 2, 4, 8 bands (rfx_group_create_inprocess, one context) render their members one after the other on one
stream, so a group's frame time is the sum of its members' kernel times.  Its ratio to the plain chain's frame time is the cost of
row-sharding on one card: the halo rows every member recomputes, and the history rows read on their owners.  Setups are timed with CUDA events in alternating blocks.  Before the timed region every group's outputs are compared with the
plain chain's byte for byte (self_check)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import chain_harness as ch  # noqa: E402
from bench_ao import device_info  # noqa: E402
from realism_effects_b200 import abi, engine, parallel  # noqa: E402

WORKLOADS = {"ssr_full_temporal": ch.Opts(mode=abi.MODE_SSR, denoise_mode=1), "ssgi_full_temporal": ch.Opts(denoise_mode=1)}
OUTPUTS = {"ssr_full_temporal": (0, 1, 2), "ssgi_full_temporal": (0, 1, 2, 3)}
WORLDS = (2, 4, 8)


def one_gpu(a, name) -> dict:
    import torch

    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda", reference_env=True)
    ctx = engine.Context(0, inp.blue)
    ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    copt = ch.chain_options(inp, WORKLOADS[name])
    plain = engine.SsgiChain(ctx, copt)
    groups = {n: parallel.InProcessGroup(ctx, copt, n) for n in WORLDS}
    frames = [([ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")], abi.make_camera(fr["cam"]), fr) for fr in inp.frames]
    count = {s: 0 for s in ("plain", *WORLDS)}

    def step(s):
        planes, cam, fr = frames[count[s] % len(frames)]
        moved = count[s] > 0
        if s == "plain":
            plain.render(cam, *planes, fr["cam"]["position"], moved)
        else:  # no per-frame host wait: one stream orders the members and the frames
            groups[s].render(cam, *planes, fr["cam"]["position"], moved, wait=False)
        count[s] += 1

    check = {}
    for i in range(a.warmup):
        for s in count:
            step(s)
        if i in (0, a.warmup - 1):  # bit-exact against the plain chain before the timed region
            ctx.sync()
            for n in WORLDS:
                ok = all(plain.download(w).tobytes() == groups[n].download(w).tobytes() for w in OUTPUTS[name])
                check[f"n{n}"] = check.get(f"n{n}", True) and ok
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
    res = {"workload": f"{name} at {W}x{H}, demo HDR env, one chain vs in-process groups on one GPU", "frames": nf, "warmup": a.warmup,
           "self_check_bit_exact": check, "ms_plain": round(per["plain"], 4)}
    for n in WORLDS:
        res[f"ms_group_n{n}_sum_of_members"] = round(per[n], 4)
        res[f"overhead_n{n}"] = round(per[n] / per["plain"], 4)
    for g in groups.values():
        g.close()
    plain.close()
    ctx.close()
    return res


def multi_gpu(a, rank, world, name, W, H) -> dict:
    """W x H row-sharded over `world` GPUs (one process each): ms per frame of every rank"""
    import torch
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    inp = ch.make_inputs(W, H, 2, device="cuda", reference_env=True)
    ctx = engine.Context(rank, inp.blue)
    ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", rank))
    sh = parallel.ShardedSsgiChain(ctx, ch.chain_options(inp, WORKLOADS[name]))
    frames = [([ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")], abi.make_camera(fr["cam"]), fr) for fr in inp.frames]
    for i in range(a.warmup):
        planes, cam, fr = frames[i % 2]
        sh.render(cam, *planes, fr["cam"]["position"], i > 0)
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(a.frames):
        planes, cam, fr = frames[i % 2]
        sh.render(cam, *planes, fr["cam"]["position"], True)
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

    assert torch.cuda.is_available(), "bench_group_modes.py measures on the GPU; there is no CPU timing"
    assert a.frames >= 100 and a.warmup >= 2, "at least 100 timed frames and 2 warm-up frames"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    res = {"device": device_info(rank)}
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("gloo")
        for name in WORKLOADS:
            res[f"{name}_sharded"] = multi_gpu(a, rank, world, name, a.width, a.height)
            res[f"{name}_c5"] = multi_gpu(a, rank, world, name, 7680, 4320)
        dist.destroy_process_group()
    if rank == 0:
        for name in WORKLOADS:
            res[name] = one_gpu(a, name)
        print(json.dumps(res))


if __name__ == "__main__":
    main()
