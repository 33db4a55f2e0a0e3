"""The cosmetic stage of the TRAA tail (rfx_*_chain_set_effects: `EffectPass(camera, sharpnessEffect)` as the frame's last pass) at
3840 x 2160 on one GPU.  Prints one JSON line with the card's name and power limit.

    python tools/bench_fx_stage.py [--frames 100] [--warmup 10] [--width 3840 --height 2160]

Two workloads, each as three chains timed with CUDA events on the context's stream in alternating blocks:
  ssgi_c3   the SSGI + TRAA frame of tools/bench_traa.py (fast chain, denoiseIterations 2, TRAA tail);
  ao_c4     the AO frame of tools/bench_ao_traa.py (K6 spp 8, iterations 1, K7, TRAA tail), and in-process groups of N = 2, 4, 8 bands with
            the stage (the members render one after the other on one card, so a group's frame is the sum of its members' kernel times and its
            ratio to the chain with the stage is the cost of sharding);
against each other: the chain with the tail, the chain with the tail and the stage (the demo's SharpnessEffect({ sharpness: 0.75 })), and the
chain with the tail followed by a separate rfx_effects_launch with the same values.  Before the timed region the stage's output is checked
byte for byte against the separate launch, and every group's against the chain.  `extra_rows_per_band` gives, for N equal bands of the
frame, the mean number of rows the stage makes every band's tail recompute beyond the band: with Sharpness, and with LensDistortion at its
defaults (alphax = alphay = -0.05, aberration 1)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import chain_harness as ch  # noqa: E402
from bench_ao import device_info  # noqa: E402
from bench_mb_tail import WORLDS, _time  # noqa: E402
from realism_effects_b200 import abi, engine, parallel  # noqa: E402

SETUPS = ("tail", "stage", "separate")


def _fx(cam_u) -> abi.EffectsParams:
    return abi.make_effects_params(cam_u, [abi.FX_SHARPNESS], sharpness=0.75)  # example/main.js: new SharpnessEffect({ sharpness: 0.75 })


def ssgi_c3(a) -> dict:
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda", reference_env=True)
    ctx = engine.Context(0, inp.blue)
    ctx.set_env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    copt, topt = ch.chain_options(inp, ch.Opts(denoise_iterations=2)), abi.make_traa_tail_options()
    chains = {s: engine.SsgiChain(ctx, copt) for s in SETUPS}
    for c in chains.values():
        c.enable_traa(topt)
    frames = [([ctx.upload(fr[k]) for k in ("depth", "gbuffer", "velocity", "direct")], abi.make_camera(fr["cam"]), fr) for fr in inp.frames]
    sep = ctx.alloc(abi.FMT_RGBA16F, W, H)
    n = {s: 0 for s in chains}

    def step(s):
        planes, cam, fr = frames[n[s] % len(frames)]
        p = _fx(fr["cam"])
        if s == "stage":
            chains[s].set_effects(p)
        chains[s].render(cam, *planes, fr["cam"]["position"], n[s] > 0)
        if s == "separate":
            ctx.effects(p, chains[s].output(6), planes[0], planes[2], sep)
        n[s] += 1

    for _ in range(a.warmup):
        for s in chains:
            step(s)
    ctx.sync()
    check = {"stage_equals_separate_launch": chains["stage"].download(6).tobytes() == sep.download().tobytes(),
             "stage_input_equals_tail": chains["stage"].download(8).tobytes() == chains["separate"].download(6).tobytes()}
    per = _time(a, ctx, step, list(chains))
    for c in chains.values():
        c.close()
    ctx.close()
    return {"workload": f"SSGI C3 at {W}x{H}, denoiseIterations 2, TRAA tail; Sharpness 0.75", "frames": a.frames, "warmup": a.warmup,
            "self_check_bit_exact": check, "ms_chain_with_tail": round(per["tail"], 4), "ms_chain_with_tail_and_stage": round(per["stage"], 4),
            "ms_chain_with_tail_and_separate_launch": round(per["separate"], 4), "ms_stage": round(per["stage"] - per["tail"], 4)}


def ao_c4(a) -> dict:
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda")
    ctx = engine.Context(0, inp.blue)
    copt, topt = engine.ao_chain_options(W, H, {"iterations": 1}), abi.make_traa_tail_options()
    chains = {s: engine.AoChain(ctx, copt) for s in SETUPS}
    for c in chains.values():
        c.enable_traa(topt)
    frames = [(ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"]), fr["cam"]) for fr in inp.frames]
    groups = {w: parallel.InProcessAoGroup(ctx, copt, w, traa=topt) for w in WORLDS}
    setups = [*chains, *groups]
    outs = {s: ctx.alloc(abi.FMT_RGBA16F, W, H) for s in setups}
    sep = ctx.alloc(abi.FMT_RGBA16F, W, H)
    n = {s: 0 for s in setups}

    def step(s):
        d, v, i, u = frames[n[s] % len(frames)]
        p = _fx(u)
        if s in groups:  # no per-frame host wait: one stream orders the members and the frames
            groups[s].set_effects(p)
            groups[s].render(u, d, v, None, i, outs[s], wait=False, traa_cam=u, camera_moved=True)
        else:
            if s == "stage":
                chains[s].set_effects(p)
            chains[s].render(u, d, v, None, i, outs[s], traa_cam=u, camera_moved=True)
            if s == "separate":
                ctx.effects(p, outs[s], d, v, sep)
        n[s] += 1

    for _ in range(a.warmup):
        for s in setups:
            step(s)
    ctx.sync()
    check = {"stage_equals_separate_launch": outs["stage"].download().tobytes() == sep.download().tobytes()}
    for w, g in groups.items():
        check[f"group_n{w}"] = outs[w].download().tobytes() == outs["stage"].download().tobytes()
    per = _time(a, ctx, step, setups)
    for g in groups.values():
        g.close()
    for c in chains.values():
        c.close()
    ctx.close()
    return {"workload": f"AO C4 (K6 spp 8) at {W}x{H}, iterations 1, K7, TRAA tail; Sharpness 0.75", "frames": a.frames, "warmup": a.warmup,
            "self_check_bit_exact": check, "ms_chain_with_tail": round(per["tail"], 4), "ms_chain_with_tail_and_stage": round(per["stage"], 4),
            "ms_chain_with_tail_and_separate_launch": round(per["separate"], 4), "ms_stage": round(per["stage"] - per["tail"], 4),
            **{f"ms_group_n{w}_sum_of_members": round(per[w], 4) for w in WORLDS},
            **{f"overhead_n{w}": round(per[w] / per["stage"], 4) for w in WORLDS}}


def extra_rows(W: int, H: int) -> dict:
    """mean rows beyond its band that the stage makes each of N equal bands recompute (host arithmetic: parallel.fx_stage_rows)"""
    res = {}
    for name, ids in (("sharpness", [abi.FX_SHARPNESS]), ("lens_distortion_defaults", [abi.FX_LENS_DISTORTION])):
        for w in WORLDS:
            b = [H * i // w for i in range(w + 1)]
            extra = [(lambda r: r[1] - r[0])(parallel.fx_stage_rows(W, H, (b[k], b[k + 1]), ids)) - (b[k + 1] - b[k]) for k in range(w)]
            res[f"{name}_n{w}"] = round(sum(extra) / w, 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_fx_stage.py measures on the GPU; there is no CPU timing"
    assert a.frames >= 100 and a.warmup >= 2, "at least 100 timed frames and 2 warm-up frames"
    res = {"device": device_info(0), "ssgi_c3": ssgi_c3(a), "ao_c4": ao_c4(a), "extra_rows_per_band": extra_rows(a.width, a.height)}
    res["self_check_passed"] = all(all(res[k]["self_check_bit_exact"].values()) for k in ("ssgi_c3", "ao_c4"))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
