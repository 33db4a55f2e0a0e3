"""The SSGI + TRAA frame (BASELINE.json C3: SSGI + TRAA + PoissonDenoise at 3840 x 2160 on one GPU) with the chain's TRAA tail, on the
bench.py workload (synthetic scene, demo HDR environment, denoiseIterations 2).  Prints one JSON line.

    python tools/bench_traa.py [--frames 100] [--warmup 10] [--width 3840 --height 2160]
    python -m torch.distributed.run --nproc_per_node N tools/bench_traa.py     # + C5: 7680 x 4320 row-sharded over N GPUs with the tail

Two setups, each on its own chain, timed in alternating blocks in one process (CUDA events on the context's stream):
  (a) the chain alone;  (b) the chain with its TRAA tail (ssgi_compose -> temporal_reproject in its TRAA form -> traa_compose).
Reported: ms per frame of each, the tail's cost (b - a), Mpx/s of (b) with the 540 B/px algorithmic traffic of the frame (BASELINE.md:
432 for the chain, then K5, the 1-plane TRAA form of K2 and K9) and its share of the H100 SXM data-sheet 3.35 TB/s, and the card's name
and power limit.  tests/test_gpu_traa_tail.py holds the tail's bytes to the stand-alone launches."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import chain_harness as ch  # noqa: E402
from bench_ao import device_info  # noqa: E402
from realism_effects_b200 import abi, engine  # noqa: E402

BYTES_PER_PX = 540
HBM_PEAK = 3.35e12  # H100 SXM data sheet


def single_gpu(a) -> dict:
    import torch

    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda", reference_env=True)
    o = ch.Opts(denoise_iterations=2)
    ctx = engine.Context(0, inp.blue)
    ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    copt = ch.chain_options(inp, o)
    topt = abi.make_traa_tail_options()
    chains = {s: engine.SsgiChain(ctx, copt) for s in "ab"}
    chains["b"].enable_traa(topt)
    frames = [([ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")], abi.make_camera(fr["cam"]), fr) for fr in inp.frames]
    n = {s: 0 for s in "ab"}

    def step(s):
        planes, cam, fr = frames[n[s] % len(frames)]
        chains[s].render(cam, *planes, fr["cam"]["position"], n[s] > 0)
        n[s] += 1

    for s in "ab":
        for _ in range(a.warmup):
            step(s)
    ctx.sync()
    blocks = 4
    ms = {s: 0.0 for s in "ab"}
    for _ in range(blocks):  # alternate the setups so that clock and neighbour load drift hit both alike
        for s in "ab":
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.frames // blocks):
                step(s)
            e1.record(stream)
            e1.synchronize()
            ms[s] += e0.elapsed_time(e1)
    per = {s: ms[s] / (blocks * (a.frames // blocks)) for s in "ab"}
    mpx = W * H / (per["b"] * 1e-3) / 1e6
    res = {"c3": {"workload": f"C3 as BASELINE.json defines it: SSGI (denoiseIterations 2) + TRAA at {W}x{H}, demo HDR env", "frames": blocks * (a.frames // blocks),
                  "warmup": a.warmup, "ms_chain": round(per["a"], 4), "ms_chain_with_tail": round(per["b"], 4), "tail_ms": round(per["b"] - per["a"], 4),
                  "mpx_per_s": round(mpx, 1), "algorithmic_bytes_per_px": BYTES_PER_PX,
                  "algorithmic_share_of_3.35TBps": round(BYTES_PER_PX * W * H / (per["b"] * 1e-3) / HBM_PEAK, 4)}}
    for c in chains.values():
        c.close()
    ctx.close()
    return res


def c5(a, rank, world) -> dict:
    """7680 x 4320 row-sharded over `world` GPUs (one process each) with the tail: ms per frame of the slowest rank"""
    import torch
    import torch.distributed as dist

    from realism_effects_b200 import parallel

    W, H = 7680, 4320
    torch.cuda.set_device(rank)
    inp = ch.make_inputs(W, H, 2, device="cuda", reference_env=True)
    ctx = engine.Context(rank, inp.blue)
    ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", rank))
    sh = parallel.ShardedSsgiChain(ctx, ch.chain_options(inp, ch.Opts(denoise_iterations=2)), traa=abi.make_traa_tail_options())
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
    t = torch.tensor([e0.elapsed_time(e1) / a.frames], device=f"cuda:{rank}")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t.item())
    sh.close()
    ctx.close()
    return {"c5": {"workload": f"C5: SSGI (denoiseIterations 2) + TRAA at {W}x{H} row-sharded over {world} GPUs", "frames": a.frames, "ms_per_frame": round(ms, 4),
                   "mpx_per_s": round(W * H / (ms * 1e-3) / 1e6, 1)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_traa.py measures on the GPU; there is no CPU timing"
    assert a.frames >= 100, "at least 100 timed frames"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    res = {"device": device_info(rank)}
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("gloo")
        res.update(c5(a, rank, world))
        if rank == 0:
            res.update(single_gpu(a))
        dist.destroy_process_group()
    else:
        res.update(single_gpu(a))
    if rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
