"""The AO chain from host buffers (rfx_ao_chain_render_host / _submit_host / _wait_host) at 3840 x 2160 on one GPU.  Prints one JSON line with
the card's name and power limit.

    python tools/bench_ao_host.py [--frames 100] [--warmup 10] [--width 3840 --height 2160]

Two workloads: C4 (K6 spp 8, iterations 1, K7) and C4 with the TRAA tail (K7 -> TRAA -> K9).  Each runs three ways:
  device      rfx_ao_chain_render(_traa) on planes already on the device (kernels only);
  render_host one frame in, its result out: H2D of depth, velocity and the scene colour, the kernels, D2H of out_color, in sequence;
  pipelined   submit_host with one frame in flight (wait_host(1)) over two pinned host buffer sets: frame i+1 uploads and frame i-1
              downloads while frame i renders.
Every way is timed on the host clock over a window that ends in a synchronise.  The bytes per frame are computed from the plane formats
(H2D: depth 4 + velocity 16 + colour 8 B/px; D2H: out_color 8 B/px), and the effective rate is those bytes over the time per frame.
Before the timed region the three ways are checked byte for byte against each other on three moving frames."""
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

H2D_BPP, D2H_BPP = 4 + 16 + 8, 8


class Workload:
    def __init__(self, ctx, inp, W, H, tail: bool):
        import torch

        self.ctx, self.inp, self.W, self.H, self.tail = ctx, inp, W, H, tail
        self.copt = engine.ao_chain_options(W, H, {"spp": 8, "iterations": 1})
        self.dev_planes = [(ctx.upload(fr["depth"]), ctx.upload(fr["velocity"]), ctx.upload(fr["direct"])) for fr in inp.frames]
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()  # noqa: E731
        # one pinned set per input frame; the pipelined way alternates two of them, which is what a caller double-buffering does
        self.host = [dict(depth=pin(fr["depth"]), velocity=pin(fr["velocity"]), input=pin(fr["direct"]),
                          out=torch.zeros((H, W, 4), dtype=torch.float16).pin_memory()) for fr in inp.frames]
        self.out = ctx.alloc(abi.FMT_RGBA16F, W, H)

    def chain(self):
        c = engine.AoChain(self.ctx, self.copt)
        if self.tail:
            c.enable_traa()
        return c

    def cam(self, t):
        return self.inp.frames[t % len(self.inp.frames)]["cam"]

    def device(self, c, t):
        d, v, i = self.dev_planes[t % len(self.dev_planes)]
        u = self.cam(t)
        c.render(u, d, v, None, i, self.out, traa_cam=u if self.tail else None, camera_moved=True)

    def host_frame(self, c, t):
        h, u = self.host[t % len(self.host)], self.cam(t)
        return c.host_frame(u, h["depth"], h["velocity"], None, h["input"], h["out"], None, traa_cam=u if self.tail else None, camera_moved=True)

    def check(self) -> dict:
        """three frames each way on fresh chains: the same out_color bytes"""
        dev, sync, pipe = self.chain(), self.chain(), self.chain()
        want, got_sync = [], []
        for t in range(3):
            self.device(dev, t)
            want.append(self.out.download().tobytes())
            sync.render_host(self.host_frame(sync, t))
            got_sync.append(self.host[t % len(self.host)]["out"].numpy().tobytes())
        hfs, got_pipe = [], []
        for t in range(3):
            hfs.append(self.host_frame(pipe, t))
            pipe.submit_host(hfs[-1])
            pipe.wait_host(1)
            if t >= 1:  # frame t-1 is complete; its set is reused by frame t+1
                got_pipe.append(self.host[(t - 1) % len(self.host)]["out"].numpy().tobytes())
        pipe.wait_host(0)
        got_pipe.append(self.host[2 % len(self.host)]["out"].numpy().tobytes())
        for c in (dev, sync, pipe):
            c.close()
        return {"render_host_equals_device": got_sync == want, "pipelined_equals_device": got_pipe == want}

    def time(self, frames: int, warmup: int) -> dict:
        res = {}
        for way in ("device", "render_host", "pipelined"):
            c = self.chain()
            hfs = [self.host_frame(c, t) for t in range(len(self.host))]

            def run(n, t0):
                for t in range(t0, t0 + n):
                    if way == "device":
                        self.device(c, t)
                    elif way == "render_host":
                        c.render_host(hfs[t % len(hfs)])
                    else:
                        c.submit_host(hfs[t % len(hfs)])
                        c.wait_host(1)
                if way == "device":
                    self.ctx.sync()
                else:
                    c.wait_host(0)

            run(warmup, 0)
            t0 = time.perf_counter()
            run(frames, warmup)
            res[way] = (time.perf_counter() - t0) * 1e3 / frames
            c.close()
        px = self.W * self.H
        h2d, d2h = H2D_BPP * px, D2H_BPP * px
        out = {f"ms_{w}": round(ms, 4) for w, ms in res.items()}
        out.update(h2d_bytes_per_frame=h2d, d2h_bytes_per_frame=d2h,
                   **{f"GBps_{w}": round((h2d + d2h) / (res[w] * 1e-3) / 1e9, 2) for w in ("render_host", "pipelined")})
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_ao_host.py measures on the GPU; there is no CPU timing"
    W, H = a.width, a.height
    inp = ch.make_inputs(W, H, 2, device="cuda")
    ctx = engine.Context(0, inp.blue)
    res = {"device": device_info(0)}
    for name, tail in (("ao_c4", False), ("ao_c4_traa", True)):
        w = Workload(ctx, inp, W, H, tail)
        res[name] = {"workload": f"AO C4 (K6 spp 8) at {W}x{H}, iterations 1, K7" + (", TRAA tail" if tail else ""), "frames": a.frames,
                     "warmup": a.warmup, "self_check_bit_exact": w.check(), **w.time(a.frames, a.warmup)}
    res["self_check_passed"] = all(all(res[k]["self_check_bit_exact"].values()) for k in ("ao_c4", "ao_c4_traa"))
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
