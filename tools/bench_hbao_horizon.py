"""C4 as the brief states it (HorizonAOEffect: K6h horizon march 8 directions x 32 steps -> 2 one-plane Poisson passes -> K7 ao_compose)
at 3840 x 2160, K6h alone, and for comparison the spp-8 C4 of HBAOEffect (K6) in the same process.  Prints one JSON line.

    python tools/bench_hbao_horizon.py [--frames 200] [--warmup 20] [--rounds 2] [--width 3840 --height 2160] [--no-parity]

Before any timing, K6h's output (both variants) is checked against the CPU oracle (tests/horizon_oracle.cpp): the fraction of pixels
outside 1e-3 relative.  Times are CUDA events on the context's stream around `frames` launches after `warmup`, repeated `rounds` times
with the variants alternating, so the spread is visible.  Tap throughput is D * S * W * H over K6h's time; its algorithmic bytes (12 B per
pixel: the depth texel and the RGBA16F output, as K6) say nothing about a gather served by the caches, so no bandwidth is derived.
The card's name and power limit are part of the line."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import ao_harness as ao  # noqa: E402
import chain_harness as ch  # noqa: E402
import horizon_harness as hz  # noqa: E402
from bench_ao import device_info, time_ms  # noqa: E402
from realism_effects_b200 import abi, engine  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--directions", type=int, default=8)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--no-parity", action="store_true")
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_hbao_horizon.py measures on the GPU; there is no CPU timing"
    assert a.frames >= 200, "at least 200 timed frames"
    W, H, D, S = a.width, a.height, a.directions, a.steps
    inp = ch.make_inputs(W, H, 1, device="cuda")
    fr = inp.frames[0]
    ctx = engine.Context(0, inp.blue)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    d, v, dl = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])
    target, tA, tB, outp = (ctx.alloc(abi.FMT_RGBA16F, W, H) for _ in range(4))
    pps = []
    for i in range(2):
        p = ch.poisson_params(ch.Opts(), 1234568 + i, False)
        p.texture_count, p.gbuffer_texture, p.input_linear = 1, 0, 1
        p.is_texture_specular[:] = [0, 0]
        p.normal_phi, p.depth_phi, p.roughness_phi, p.specular_phi = 3.25, 2.0, 0.0, 0.0
        pps.append(p)
    acp = ch.ao_compose_params()
    hzp = hz.horizon_params(fr["cam"], 778, D, S)
    hbp = ao.hbao_params(fr["cam"], 778)
    res = {"workload": f"C4 {W}x{H}: K6h {D} directions x {S} steps + 2 one-plane Poisson passes + ao_compose; K6h alone; "
                       f"HBAOEffect's C4 (K6 spp 8) for comparison",
           "frames": a.frames, "warmup": a.warmup, "rounds": a.rounds, "device": device_info(0)}

    k6h = lambda: ctx.hbao_horizon(hzp, d, target)  # noqa: E731
    k6 = lambda: ctx.hbao(hbp, d, target)  # noqa: E731

    def tail():
        ctx.poisson_denoise(pps[0], d, v, target, None, tA, None)
        ctx.poisson_denoise(pps[1], d, v, tA, None, tB, None)
        ctx.ao_compose(acp, d, tB, dl, outp)

    def c4_literal():
        k6h()
        tail()

    def c4_spp8():
        k6()
        tail()

    if not a.no_parity:
        want = hz.oracle_hbao_horizon(hzp, fr["depth"], inp.blue, np.zeros((H, W, 4), np.float16))
        for fast in (False, True):
            ctx.set_fast_math(fast)
            target.upload(np.zeros((H, W, 4), np.float16))
            k6h()
            c = ch.compare(want, target.download())
            res[f"k6h_parity_{'fast' if fast else 'exact'}"] = {"frac_bad_1e3": c["frac_bad"], "bit_equal": c["bit_equal"]}
    ctx.set_fast_math(True)
    variants = {"c4_literal": c4_literal, "k6h": k6h, "c4_spp8": c4_spp8, "k6": k6}
    times = {k: [] for k in variants}
    for fn in variants.values():
        for _ in range(a.warmup):
            fn()
    for _ in range(a.rounds):
        for k, fn in variants.items():
            for _ in range(a.warmup):
                fn()
            times[k].append(round(time_ms(stream, fn, a.frames), 4))
    res["ms"] = times
    best = min(times["k6h"])
    res["k6h_taps_per_s"] = float(f"{D * S * W * H / (best * 1e-3):.4g}")
    res["k6h_ms_min"], res["c4_literal_ms_min"] = best, min(times["c4_literal"])
    for p in (d, v, dl, target, tA, tB, outp):
        p.free()
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
