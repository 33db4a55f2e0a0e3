"""The SSGI + TRAA frame (BASELINE.json C3: SSGI + TRAA + PoissonDenoise at 3840 x 2160 on one GPU) with the chain's TRAA tail, on the
bench.py workload (synthetic scene, demo HDR environment, denoiseIterations 2).  Prints one JSON line.

    python tools/bench_traa.py [--frames 100] [--warmup 10] [--width 3840 --height 2160]
    python -m torch.distributed.run --nproc_per_node N tools/bench_traa.py     # + C5: 7680 x 4320 row-sharded over N GPUs with the tail

Three setups, each on its own chain, timed in alternating blocks in one process (CUDA events on the context's stream):
  (a) the chain alone;  (b) the chain with the fused TRAA tail;  (c) the chain followed by the three per-pass tail launches
  (ssgi_compose -> temporal_reproject in its TRAA form -> traa_compose).
Reported: ms per frame of each, the tail's cost (b - a) and (c - a), Mpx/s of (b) with the 540 B/px algorithmic traffic of the frame
(BASELINE.md: 432 for the chain, then K5, the 1-plane TRAA form of K2 and K9) and its share of the H100 SXM data-sheet 3.35 TB/s, the
card's name and power limit, and whether (b) and (c) wrote identical bytes (K9 output and TRAA history) on the last frame."""
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
    chains = {s: engine.SsgiChain(ctx, copt) for s in "abc"}
    chains["b"].enable_traa(topt)
    frames = [([ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")], abi.make_camera(fr["cam"]), fr) for fr in inp.frames]
    k5, out = ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)
    acc = [ctx.alloc(abi.FMT_RGBA16F, W, H), ctx.alloc(abi.FMT_RGBA16F, W, H)]
    n = {s: 0 for s in "abc"}
    state = {"keep": 0.0, "prev": None}

    def step(s):
        planes, cam, fr = frames[n[s] % len(frames)]
        moved = n[s] > 0
        chains[s].render(cam, *planes, fr["cam"]["position"], moved)
        if s == "c":
            t = n[s]
            ctx.ssgi_compose(planes[0], chains[s].output(0), planes[3], k5, params=topt.compose)
            tp = ch.traa_temporal_params(cam, fr["cam"]["position"], state["prev"] or fr["cam"], state["keep"])
            tp.full_accumulate = int(bool(topt.full_accumulate) and not moved)
            ctx.temporal_reproject(tp, k5, planes[2], acc[(t + 1) & 1], None, acc[t & 1], None)
            ctx.traa_compose(acc[t & 1], out)
            state["keep"], state["prev"] = 1.0, fr["cam"]
        n[s] += 1

    for s in "abc":
        for _ in range(a.warmup):
            step(s)
    ctx.sync()
    blocks = 4
    ms = {s: 0.0 for s in "abc"}
    for _ in range(blocks):  # alternate the setups so that clock and neighbour load drift hit all three alike
        for s in "abc":
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.frames // blocks):
                step(s)
            e1.record(stream)
            e1.synchronize()
            ms[s] += e0.elapsed_time(e1)
    per = {s: ms[s] / (blocks * (a.frames // blocks)) for s in "abc"}
    identical = (chains["b"].download(6).tobytes() == out.download().tobytes() and chains["b"].download(7).tobytes() == acc[(n["c"] - 1) & 1].download().tobytes()
                 and n["b"] == n["c"])
    mpx = W * H / (per["b"] * 1e-3) / 1e6
    res = {"c3": {"workload": f"C3 as BASELINE.json defines it: SSGI (denoiseIterations 2) + TRAA at {W}x{H}, demo HDR env", "frames": blocks * (a.frames // blocks),
                  "warmup": a.warmup, "ms_chain": round(per["a"], 4), "ms_chain_fused_tail": round(per["b"], 4), "ms_chain_per_pass_tail": round(per["c"], 4),
                  "tail_ms_fused": round(per["b"] - per["a"], 4), "tail_ms_per_pass": round(per["c"] - per["a"], 4),
                  "mpx_per_s_fused": round(mpx, 1), "algorithmic_bytes_per_px": BYTES_PER_PX,
                  "algorithmic_share_of_3.35TBps": round(BYTES_PER_PX * W * H / (per["b"] * 1e-3) / HBM_PEAK, 4),
                  "fused_equals_per_pass_last_frame": identical}}
    for c in chains.values():
        c.close()
    ctx.close()
    return res


def c5(a, rank, world) -> dict:
    """7680 x 4320 row-sharded over `world` GPUs (one process each) with the fused tail: ms per frame of the slowest rank"""
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
