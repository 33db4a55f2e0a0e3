"""GPU box: oracle-vs-CUDA parity of the SSGI chain at the BASELINE config sizes (C2 1920x1080, C3 3840x2160), both kernel
variants, >= 3 frames with history.  Writes one JSON document (per frame, per plane: fraction of pixels outside 1e-3 / 4e-3
relative, max relative error of the conforming pixels, bit-equality, and how many pixels' bytes differ, with the first one).  TEST INFRASTRUCTURE (runs the oracle).
usage: python tools/parity_at_size.py [C2] [C3] [--frames N] [--out gpurun_out/parity_at_size.json]"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import chain_harness as ch  # noqa: E402

CONFIGS = {"C2": dict(width=1920, height=1080, denoise_iterations=1), "C3": dict(width=3840, height=2160, denoise_iterations=2),
           "tiny": dict(width=192, height=108, denoise_iterations=1)}
PLANES = ("ssgi", "tr0", "tr1", "dn0", "dn1", "composed")


def differing_pixels(a, b):
    """(y, x) of the pixels whose bytes differ; in an fp16 plane a channel NaN on both sides counts as equal (as
    tests/chain_harness.differing_pixels, which says why)"""
    import numpy as np

    u = {2: np.uint16, 4: np.uint32}[a.dtype.itemsize]
    d = a.view(u) != b.view(u)
    if a.dtype == np.float16:
        d &= ~(np.isnan(a) & np.isnan(b))
    return np.argwhere(d.reshape(a.shape[0], a.shape[1], -1).any(-1))


def run(name, frames, variants=(True, False)):
    kw = dict(CONFIGS[name])
    W, H = kw.pop("width"), kw.pop("height")
    o = ch.Opts(**kw)
    t0 = time.perf_counter()
    inp = ch.make_inputs(W, H, frames, env_size=(1024, 512) if W >= 1920 else (128, 64))
    t1 = time.perf_counter()
    ref = ch.run_oracle_chain(inp, o, lean=True)
    t2 = time.perf_counter()
    res = {"config": name, "width": W, "height": H, "frames": frames, "denoise_iterations": o.denoise_iterations, "synth_s": round(t1 - t0, 1),
           "oracle_s": round(t2 - t1, 1), "variants": {}}
    for fast in variants:
        got, launches = ch.run_cuda_chain(inp, o, fast_math=fast)
        rows = []
        for t in range(frames):
            for k in PLANES:
                c = ch.compare(ref[t][k], got[t][k], packed=(k == "ssgi"))
                c4 = ch.compare(ref[t][k], got[t][k], packed=(k == "ssgi"), rtol=4e-3)
                d = differing_pixels(ref[t][k], got[t][k])
                rows.append(dict(frame=t, plane=k, frac_bad_1e3=c["frac_bad"], n_bad=c["n_bad"], frac_bad_4e3=c4["frac_bad"], max_rel_ok=c["max_rel_ok"],
                                 max_abs=c["max_abs"], bit_equal=c["bit_equal"], n_differ=len(d), first_differ=[int(v) for v in d[0]] if len(d) else None))
        res["variants"]["fast" if fast else "exact"] = dict(launches=launches, worst_frac_bad_1e3=max(r["frac_bad_1e3"] for r in rows),
                                                           worst_frac_bad_4e3=max(r["frac_bad_4e3"] for r in rows), rows=rows)
        del got
    return res


if __name__ == "__main__":
    args = sys.argv[1:]
    frames, out = 3, os.path.join(ROOT, "gpurun_out", "parity_at_size.json")
    names = [a for a in args if a in CONFIGS] or ["C2", "C3"]
    if "--frames" in args:
        frames = int(args[args.index("--frames") + 1])
    if "--out" in args:
        out = args[args.index("--out") + 1]
    doc = []
    for n in names:
        r = run(n, frames, (True,) if "--fast-only" in args else (True, False))
        doc.append(r)
        for v, d in r["variants"].items():
            print(f"{n} {v}: worst frac_bad@1e-3 {d['worst_frac_bad_1e3']:.3e}  @4e-3 {d['worst_frac_bad_4e3']:.3e}  (oracle {r['oracle_s']} s)")
            for row in d["rows"]:
                print(f"   f{row['frame']}.{row['plane']:9s} bad {row['frac_bad_1e3']:.2e} ({row['n_bad']}) bad@4e-3 {row['frac_bad_4e3']:.1e} max_rel_ok {row['max_rel_ok']:.1e} biteq {row['bit_equal']:.5f} differ {row['n_differ']}")
        sys.stdout.flush()
    os.makedirs(os.path.dirname(out), exist_ok=True)
    json.dump(doc, open(out, "w"), indent=1)
