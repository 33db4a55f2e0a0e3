"""C4 (HBAOEffect: K6 HBAO spp 8 -> 2 one-plane Poisson passes -> K7 ao_compose) at 3840 x 2160 and resolutionScale 1, 0.75 and 0.5,
with depth-rebuilt normals and with a normal plane (useNormalPass / normalTexture).  Prints one JSON line.

    python tools/bench_ao.py [--frames 200] [--warmup 10] [--width 3840 --height 2160] [--no-parity]

Per variant: device ms per C4 frame and K6's own ms (CUDA events on the context's stream around `frames` launches after `warmup`),
and the parity of the first frame's K6 output against the CPU oracle (fraction of pixels outside 1e-3 relative; the denoise and compose
at reduced scale are checked by tests/test_gpu_ao_scale.py).  The card's name and power limit are part of the line.
The Poisson passes and the compose run at full size whatever the scale, so only K6's share of C4 shrinks with the scale."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import ao_harness as ao  # noqa: E402
import chain_harness as ch  # noqa: E402
from realism_effects_b200 import abi, engine  # noqa: E402


def device_info(gpu_index: int) -> dict:
    import torch

    info = {"name": torch.cuda.get_device_name(gpu_index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(gpu_index)],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip())
    except Exception:  # noqa: BLE001
        pass
    return info


def time_ms(stream, fn, n):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--no-parity", action="store_true")
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_ao.py measures on the GPU; there is no CPU timing"
    assert a.frames >= 100, "at least 100 timed frames"
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 1, device="cuda")
    fr = inp.frames[0]
    normal_host = ao.view_normal_plane(W, H, 0, fr["cam"])
    ctx = engine.Context(0, inp.blue)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    d, v, dl, nrm = ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"]), ctx.upload(normal_host)
    tA, tB, outp = (ctx.alloc(abi.FMT_RGBA16F, W, H) for _ in range(3))
    pps = []
    for i in range(2):
        p = ch.poisson_params(ch.Opts(), 1234568 + i, False)
        p.texture_count, p.gbuffer_texture, p.input_linear = 1, 0, 1
        p.is_texture_specular[:] = [0, 0]
        p.normal_phi, p.depth_phi, p.roughness_phi, p.specular_phi = 3.25, 2.0, 0.0, 0.0
        pps.append(p)
    acp = ch.ao_compose_params()
    res = {"workload": f"C4 {W}x{H}: HBAO spp 8 on the scaled AO target + 2 one-plane Poisson passes + ao_compose at full size",
           "frames": a.frames, "warmup": a.warmup, "device": device_info(0), "variants": {}}
    for scale in (1.0, 0.75, 0.5):
        (tw, th), resolution = ao.ao_target_size(W, H, scale)
        target = ctx.alloc(abi.FMT_RGBA16F, tw, th)
        hp = ao.hbao_params(fr["cam"], 778)
        hp.resolution[:] = list(resolution)
        for normals in ("depth", "normal_plane"):
            n = nrm if normals == "normal_plane" else None
            k6 = lambda: ctx.hbao(hp, d, target, normal=n)  # noqa: E731

            def c4():
                k6()
                ctx.poisson_denoise(pps[0], d, v, target, None, tA, None)
                ctx.poisson_denoise(pps[1], d, v, tA, None, tB, None)
                ctx.ao_compose(acp, d, tB, dl, outp)

            ctx.sync()
            c4()
            row = {"ao_target": [tw, th], "resolution": list(resolution)}
            if not a.no_parity:
                want = ao.oracle.hbao(hp, fr["depth"], inp.blue, np.zeros((th, tw, 4), np.float16), out_size=(tw, th),
                                      normal=normal_host if n is not None else None, resolution=resolution)
                row["k6_parity_frac_bad_1e3"] = ch.compare(want, target.download())["frac_bad"]
            for _ in range(a.warmup):
                c4()
            row["c4_ms"] = round(time_ms(stream, c4, a.frames), 4)
            for _ in range(a.warmup):
                k6()
            row["k6_ms"] = round(time_ms(stream, k6, a.frames), 4)
            res["variants"][f"scale_{scale}_{normals}"] = row
        target.free()
    for p in (d, v, dl, nrm, tA, tB, outp):
        p.free()
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
