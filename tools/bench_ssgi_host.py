"""The SSGI chain's compose stage (rfx_ssgi_chain_set_compose) and its image through host buffers at 3840 x 2160 on one GPU.  Prints one JSON
line with the card's name and power limit.

    python tools/bench_ssgi_host.py [--frames 60] [--warmup 10] [--rounds 3] [--width 3840 --height 2160]

Workload C3: steps 20, refineSteps 5, denoiseIterations 2 (the fast chain), Fog.  Two comparisons, each way alternated over `rounds` rounds
(min and max of the rounds are reported, so the spread is visible):
  device   the chain with the fused stage (K5 in K4's epilogue, output 9) against the chain followed by a separate rfx_ssgi_compose_launch
           over output 0, on planes already on the device: a host clock over `frames` frames that ends in a synchronise;
  host     render_host and pipelined submit_host / wait_host(1) over two pinned host sets, with out_color only (the RGBA16F image, 8 B/px
           D2H) against out_composed only (RGBA32F, 16 B/px D2H).  H2D is depth 4 + gbuffer 16 + velocity 16 + direct light 8 B/px.
Before the timed region the fused image is checked byte for byte against the separate launch, and the host ways against the device planes."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

import chain_harness as ch  # noqa: E402
from bench_ao import device_info  # noqa: E402
from realism_effects_b200 import abi, engine  # noqa: E402

H2D_BPP = 4 + 16 + 16 + 8
IN = ("depth", "gbuffer", "velocity", "direct")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_ssgi_host.py measures on the GPU; there is no CPU timing"
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda")
    ctx = engine.Context(0, inp.blue)
    ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    copt = ch.chain_options(inp, ch.Opts(denoise_iterations=2))
    fog = [ch.fog_params(fr["cam"], False) for fr in inp.frames]
    dev = [[ctx.upload(fr[k]) for k in IN] for fr in inp.frames]
    sep_out = ctx.alloc(abi.FMT_RGBA16F, W, H)
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory()  # noqa: E731
    host = [{k: pin(fr[k]) for k in IN} for fr in inp.frames]
    outs = [(torch.zeros((H, W, 4), dtype=torch.float32).pin_memory(), torch.zeros((H, W, 4), dtype=torch.float16).pin_memory()) for _ in inp.frames]
    n = len(inp.frames)

    def chain(fused: bool):
        c = engine.SsgiChain(ctx, copt)
        if fused:
            c.set_compose(fog[0])
        return c

    def device_frame(c, t, fused):
        fr, fp = inp.frames[t % n], dev[t % n]
        c.render(abi.make_camera(fr["cam"]), *fp, fr["cam"]["position"], True)
        if not fused:
            ctx.ssgi_compose(fp[0], c.output(0), fp[3], sep_out, params=fog[t % n])

    def host_frame(c, t, color):
        fr, h, o = inp.frames[t % n], host[t % n], outs[t % n]
        return c.host_frame(abi.make_camera(fr["cam"]), *(h[k] for k in IN), fr["cam"]["position"], True,
                            None if color else o[0], o[1] if color else None)

    # ---- self-check: the fused image is the separate launch's; the host ways download the device planes
    fused, sep = chain(True), chain(False)
    check = {"fused_equals_separate": True, "host_equals_device": True}
    sync = chain(True)
    for t in range(3):
        device_frame(fused, t, True)
        device_frame(sep, t, False)
        want = fused.download(9)
        check["fused_equals_separate"] &= want.tobytes() == sep_out.download().tobytes()
        sync.render_host(host_frame(sync, t, True))
        check["host_equals_device"] &= outs[t % n][1].numpy().tobytes() == want.tobytes()
    for c in (fused, sep, sync):
        c.close()

    def timed(run_frames) -> float:
        run_frames(a.warmup, 0)
        t0 = time.perf_counter()
        run_frames(a.frames, a.warmup)
        return (time.perf_counter() - t0) * 1e3 / a.frames

    res = {k: [] for k in ("device_fused", "device_separate", "render_host_color", "render_host_composed", "pipelined_color", "pipelined_composed")}
    for _ in range(a.rounds):
        for fused_way in (True, False):
            c = chain(fused_way)

            def run(k, t0, c=c, fw=fused_way):
                for t in range(t0, t0 + k):
                    device_frame(c, t, fw)
                ctx.sync()

            res["device_fused" if fused_way else "device_separate"].append(timed(run))
            c.close()
        for color in (True, False):
            for way in ("render_host", "pipelined"):
                c = chain(True)
                hfs = [host_frame(c, t, color) for t in range(n)]

                def run(k, t0, c=c, way=way, hfs=hfs):
                    for t in range(t0, t0 + k):
                        if way == "render_host":
                            c.render_host(hfs[t % n])
                        else:
                            c.submit_host(hfs[t % n])
                            c.wait_host(1)
                    c.wait_host(0)

                res[f"{way}_{'color' if color else 'composed'}"].append(timed(run))
                c.close()
    px = W * H
    out = {"device": device_info(0), "workload": f"C3 (steps 20, refineSteps 5, denoiseIterations 2, Fog) at {W}x{H}, fast chain",
           "frames": a.frames, "warmup": a.warmup, "rounds": a.rounds, "self_check_bit_exact": check,
           "h2d_bytes_per_frame": H2D_BPP * px, "d2h_bytes_per_frame": {"color": 8 * px, "composed": 16 * px}}
    for k, v in res.items():
        out[f"ms_{k}"] = {"min": round(min(v), 4), "max": round(max(v), 4)}
    for q in [p for fp in dev for p in fp] + [sep_out]:
        q.free()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
