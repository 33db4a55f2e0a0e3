"""Row-band sharding of the SSGI chain and the AO chain across N GPUs (one process per GPU).

The product path is native: `rfx_group_*` / `rfx_ssgi_chain_render_sharded` in csrc/rfx_group.inl (C ABI, include/rfx.h).
This module is the Python host binding of that API (`ShardedSsgiChain`, `ShardedAoChain`, and `InProcessGroup` / `InProcessAoGroup`
for the members of one process) plus a pure-Python mirror of its host arithmetic that the CPU tests check against the exported C
functions and drive with the oracle as compute (tests/test_sharding_cpu.py).  Every rank owns one contiguous row band.  `ShardPlan`
and `AoShardPlan` give the row range of every launch of a frame for that band (`rfx_shard_ranges` / `rfx_ao_shard_ranges`): the last
launch runs on the band, every launch before it on the next one's rows widened by what that one reads around them.

Every kernel of the path writes disjoint output rows, so the produced planes are partitioned by row band (SURVEY.md §8e).
Two kinds of inputs cross band borders:

  * bounded stencils — K2's 5x5 neighbourhood of ssgiOut (2 rows), K3's Poisson taps (ceil(radius * max(1, H/W)) + 1 rows per
    pass: the tap offset is rotated AFTER the division by the resolution, so portrait frames reach further in rows), K4's
    pixel-centre fetch (1 row).  Instead of one halo exchange per pass, each rank RECOMPUTES the halo rows itself: pass k is
    launched on a row range widened by the halos of all the passes after it.  Kernels are bit-identical under row sharding,
    so the recomputed rows equal the owner's rows bit for bit and no per-pass latency is paid (~3 % extra rows at 4K / 8 ranks).
  * arbitrary-uv gathers — K1 samples last frame's `composed` at ray hit points and K2 samples the `dn` history at reprojected
    uvs anywhere on screen.  Round 1 replicated those planes with an all-gather (32 B/px x the whole frame per rank per frame,
    which bounded the 8-GPU frame).  Now every rank keeps only its own rows and the kernels read a row another rank owns IN
    PLACE over NVLink through CUDA-IPC peer mappings (PeerPV in csrc/rfx_kernels.h); the planes are double-buffered by frame
    parity so no rank overwrites rows a peer may still read, and the frame ends with ONE tiny NCCL all-gather (each rank's
    device-timed kernel cost) that is also the frame barrier.

Adaptive bands: every few frames the borders move towards equal device-timed cost (`rfx_shard_rebalance`, mirrored by
`rebalance`: cost per row piecewise constant over the measured bands, damped, 16-row aligned; every rank derives the
same borders from the same gathered times).  All cross-frame state lives in the peer-readable planes, so borders move freely
between frames and the result stays bit-identical to the single-GPU chain (tests/test_gpu_multi.py).
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass

import numpy as np


def _poisson_halo(radius: float, height: int, width: int | None) -> int:
    """rows a Poisson tap can reach: the offset is rotated after the division by the resolution (poisson_denoise.frag:183-189), so the row
    reach is radius * max(1, H / W); + 1 for the bilinear footprint / the quad-derivative helper row"""
    stretch = max(1.0, height / width) if width else 1.0
    return int(math.ceil(radius * stretch)) + 1


def _widen_back(own, height: int, reaches) -> list:
    """Row ranges [a, b) of the launches of one frame for the band `own` (mirror of widen_back in csrc/rfx_group.inl): the last launch
    runs on the band, and every launch before it on the next launch's rows widened by what that one reads around them.  reaches[k]: the
    rows launch k + 1 reads around its output rows, of what launch k wrote, so there is one launch more than reaches."""
    a, b = own
    out = [(a, b)]
    for rows in reversed(reaches):
        a, b = max(0, a - rows), min(height, b + rows)
        out.append((a, b))
    return out[::-1]


def _with_stage(own, stage_rows, height: int, reaches) -> list:
    """_widen_back for the band `own`; with the cosmetic stage (stage_rows not None) the launches are planned for stage_rows as if they were
    the band, and the stage runs on the band as one more launch (mirror of shard_ranges in csrc/rfx_group.inl)"""
    if stage_rows is None:
        return _widen_back(own, height, reaches)
    return _widen_back(tuple(stage_rows), height, reaches) + [tuple(own)]


@functools.lru_cache(maxsize=4)
def _lens_rows(width: int, height: int, alphax, alphay, aberration):
    f = np.float32
    one, two, half = f(1.0), f(2.0), f(0.5)
    W, H = f(width), f(height)
    ax, ay, ab = f(alphax), f(alphay), f(aberration)
    with np.errstate(all="ignore"):
        Y = (two * ((np.arange(height, dtype=f) + half) / H) - one)[:, None]
        X = (two * ((np.arange(width, dtype=f) + half) / W) - one)[None, :]
        r = X * X + Y * Y
        x3, y3 = X / (one - ax * r), Y / (one - ay * r)
        q = x3 * x3 + y3 * y3
        y2 = Y / (one - ay * q)
        dv = (y2 + one) * one / two
        lo = np.full(height, height, dtype=np.int64)
        hi = np.full(height, -1, dtype=np.int64)
        for d in (ab * f(0.0), ab * (one / H)):  # the v offsets of the taps: aberration * (ox, 0), aberration * (0, oy) and (ox, oy)
            fy = (dv - d) * H - half
            every = ~(np.abs(fy) < f(1.0e9))  # not finite, or beyond the kernel's saturating integer conversion: every row
            iy = np.floor(np.where(every, f(0.0), fy)).astype(np.int64)
            lo = np.minimum(lo, np.where(every, 0, np.clip(iy, 0, height - 1)).min(axis=1))
            hi = np.maximum(hi, np.where(every, height - 1, np.clip(iy + 1, 0, height - 1)).max(axis=1))
    return lo, hi


def lens_rows(width: int, height: int, alphax: float, alphay: float, aberration: float):
    """LensDistortion's rows (mirror of lens_rows in csrc/rfx_group.inl): numpy arrays lo, hi with the lowest and highest input rows the
    three taps of output row y touch.  fx_lens's uv arithmetic (csrc/k_fx.cu) in numpy float32 (IEEE, no contraction), then the bilinear
    footprint rows floor(v * H - 0.5) and the one after, clamped to the frame; a coordinate that is not finite or beyond |1e9| rows: every
    row.  Kept for the last few (size, alphax, alphay, aberration)."""
    return _lens_rows(int(width), int(height), float(np.float32(alphax)), float(np.float32(alphay)), float(np.float32(aberration)))


def fx_stage_rows(width: int, height: int, own, effects, alphax: float = -0.05, alphay: float = -0.05, aberration: float = 1.0) -> tuple:
    """Rows [a, b) of the tail's image the cosmetic stage reads for its output band `own` (mirror of rfx_fx_stage_rows): the band +- 1 row
    for every pixel's LINEAR fetch at its centre, +- 2 with Sharpness (its 3x3 LINEAR taps), and with LensDistortion every row lens_rows
    gives for the band's rows.  effects: RFX_FX_* ids (abi.FX_*); GradualBackground and Sparkle read nothing more."""
    from . import abi

    own0, own1 = int(own[0]), int(own[1])
    reach = 2 if abi.FX_SHARPNESS in effects else 1
    a, b = max(0, own0 - reach), min(height, own1 + reach)
    if abi.FX_LENS_DISTORTION in effects:
        lo, hi = lens_rows(width, height, alphax, alphay, aberration)
        a, b = min(a, int(lo[own0:own1].min())), max(b, int(hi[own0:own1].max()) + 1)
    return a, b


@dataclass
class ShardPlan:
    """Row ranges [a, b) per launch of one SSGI chain frame for the contiguous band this rank owns, in chain order: K1, K2, K3 pass 0..n-1,
    K4 and, with `traa`, the TRAA tail (mirror of rfx_shard_ranges)."""

    height: int
    world: int
    rank: int
    n_poisson_passes: int  # 2 * denoiseIterations
    radius: float
    ssgi_mode: bool = True       # as rfx_shard_ranges' ssgi_mode: the ranges do not depend on it (K4 runs in SSR mode too)
    bounds: tuple | None = None  # band borders (world + 1 ascending rows, 0 .. height); None: equal bands of height / world rows
    width: int | None = None     # frame width: portrait frames (H > W) stretch the Poisson taps' row reach by H / W
    traa: bool = False           # the TRAA tail runs as one more launch after K4 (rfx_ssgi_chain_enable_traa)
    denoise_mode: int = 0        # 0 "full"; 1 "full_temporal" / 2 "temporal" run no Poisson pass, so their ranges are those of 0 passes
    stage_rows: tuple | None = None  # the cosmetic stage (rfx_ssgi_chain_set_effects) runs on the band as one more launch after the tail,
                                     # and the chain is planned for the rows it reads (fx_stage_rows) as if they were the band

    K2_NEIGHBOURHOOD_ROWS = 2  # 5x5 clamp window (reproject.frag:57-59)
    K4_INPUT_ROWS = 1          # literal bilinear fetch of the LINEAR Poisson targets at the pixel centre
    # `composed` rows the TRAA tail reads around its band (include/rfx.h RFX_TRAA_TAIL_ROWS): 2 for the TRAA clamp window, 1 because
    # those taps are LINEAR fetches at texel centres (the reason of K4_INPUT_ROWS), 1 for K9's LINEAR fetch of the accumulated plane at
    # the pixel centre; the TRAA form takes no derivative, so no quad row
    TRAA_TAIL_ROWS = 4

    def __post_init__(self):
        if self.bounds is None:
            if self.height % self.world:
                raise ValueError(f"height {self.height} is not divisible by world size {self.world}")
            self.bounds = tuple(self.height * i // self.world for i in range(self.world + 1))
        b = tuple(int(x) for x in self.bounds)
        if len(b) != self.world + 1 or b[0] != 0 or b[-1] != self.height or any(b[i] >= b[i + 1] for i in range(self.world)):
            raise ValueError(f"bounds {b} are not {self.world + 1} ascending rows from 0 to {self.height}")
        self.bounds = b
        self.r0, self.r1 = b[self.rank], b[self.rank + 1]
        self.poisson_halo = _poisson_halo(self.radius, self.height, self.width)

    @property
    def passes(self) -> int:
        """Poisson passes the ranges are planned for: n_poisson_passes in denoiseMode "full", else none (Denoiser.js:47-52).  The native
        chain maps a full_temporal / temporal frame's K1, K2, K4 (and tail) launches onto these ranges (rfx_ssgi_chain_render_sharded)."""
        return self.n_poisson_passes if self.denoise_mode == 0 else 0

    @property
    def n_launches(self) -> int:
        return 3 + self.passes + (1 if self.traa else 0) + (1 if self.stage_rows is not None else 0)

    @property
    def ranges(self) -> list:
        n = self.passes
        # K2 reads K1's output in its 5x5 window, every Poisson pass the previous target through its taps, K4 the last Poisson target at
        # the pixel centre (nothing without a pass) and the tail `composed`.  K4 runs in both modes (SSR composes with inputType specular)
        reaches = [self.K2_NEIGHBOURHOOD_ROWS] + [self.poisson_halo] * n + [self.K4_INPUT_ROWS if n else 0]
        return _with_stage((self.r0, self.r1), self.stage_rows, self.height, reaches + ([self.TRAA_TAIL_ROWS] if self.traa else []))

    @property
    def local_input_rows(self) -> tuple:
        """Rows of the PER-PIXEL input planes (G-buffer, direct light) this rank reads: the K1 range (it contains every later launch's
        range and the rows its Poisson taps reach) + 1 row each side, because K1's literal bilinear fetch of the direct-light plane at
        the pixel centre touches row y +- 1 whenever ((y + .5) / H) * H - .5 is not exactly y.  The planes sampled at arbitrary screen
        positions (depth: ray-march taps; velocity: reprojected uv) are needed whole."""
        a, b = self.ranges[0]
        return max(0, a - 1), min(self.height, b + 1)


@dataclass
class AoShardPlan:
    """Row ranges [a, b) per launch of one AO chain frame for the band `own`, in chain order: K6 / K6h, K3 pass 0..2*iterations-1, K7
    and, with `traa`, the TRAA tail (mirror of rfx_ao_shard_ranges).  No AO pass reads a produced plane at an arbitrary uv, so the only
    cross-row reads are K7's LINEAR fetch at the pixel centre (1 row), the Poisson taps (the halo of ShardPlan) and the tail's reads of
    the K7 plane (ShardPlan.TRAA_TAIL_ROWS)."""

    width: int
    height: int
    own: tuple
    iterations: int
    radius: float
    traa: bool = False  # the TRAA tail runs as one more launch after K7 (rfx_ao_chain_enable_traa)
    stage_rows: tuple | None = None  # the cosmetic stage's input rows (fx_stage_rows), as ShardPlan.stage_rows

    K7_INPUT_ROWS = 1

    @property
    def poisson_halo(self) -> int:
        return _poisson_halo(abs(self.radius), self.height, self.width)

    @property
    def n_launches(self) -> int:
        return 2 + 2 * self.iterations + (1 if self.traa else 0) + (1 if self.stage_rows is not None else 0)

    @property
    def ranges(self) -> list:
        reaches = [self.poisson_halo] * (2 * self.iterations) + [self.K7_INPUT_ROWS] + ([ShardPlan.TRAA_TAIL_ROWS] if self.traa else [])
        return _with_stage(tuple(self.own), self.stage_rows, self.height, reaches)

    @property
    def local_input_rows(self) -> tuple:
        """Rows of the PER-PIXEL input planes (velocity, normal, input) this rank reads, for the chain without the TRAA tail: the K6 / K6h
        range (every later launch's range lies inside it) widened by the Poisson halo when there is a Poisson pass.
          * velocity: the Poisson passes read it at their pixel (and its quad partner row, y ^ 1) and at taps up to the halo away; the fast
            path decodes it once, on pass 0's range widened by the same halo (launch_gbuffer_decode).  Pass 0's range is the widest.
          * normal: K6 / K6h fetch it NEAREST at the pixel centre, which is the pixel's own row: K6's range.
          * input: K7 fetches it LINEAR at the pixel centre, which touches row y +- 1 (K7_INPUT_ROWS), and K7 runs on the band, so the rows
            are the band +- 1: inside the last Poisson pass's range, or K6's range with iterations 0.
        depth is sampled anywhere (K6 projects its samples, K6h marches up to maxRadiusPixels) and is needed whole.  With the TRAA tail the
        TRAA pass reads velocity at reprojected uvs, so this plan does not cover it."""
        a, b = self.ranges[0]
        halo = self.poisson_halo if self.iterations > 0 else 0
        return max(0, a - halo), min(self.height, b + halo)


def rebalance(bounds, costs, measured_bounds=None, align: int = 16, min_rows: int = 64, max_share: float = 4.0, damping: float = 0.6):
    """New band borders from per-rank costs (any unit) measured with `measured_bounds` (default: `bounds`).

    The cost per row is modelled as constant inside each measured band; the ideal border k is the row where the cumulative
    cost reaches k/N of the total.  The borders move `damping` of the way from `bounds` to the ideal ones (the model is coarse:
    damping avoids overshoot), are rounded to `align` rows (the kernels' tile height, so no band ends in a partial tile) and
    kept at least `min_rows` and at most max_share x the mean height apart.  Pure and deterministic: every rank computes the
    same borders from the same gathered costs."""
    mb = list(measured_bounds if measured_bounds is not None else bounds)
    n, H = len(costs), bounds[-1]
    costs = [max(float(c), 1e-9) for c in costs]
    total = sum(costs)
    ideal, k, acc = [0], 0, 0.0
    for i in range(1, n):  # invert the piecewise-linear cumulative cost at i/n of the total
        want = total * i / n
        while k < n - 1 and acc + costs[k] < want:
            acc += costs[k]
            k += 1
        ideal.append(mb[k] + (want - acc) / costs[k] * (mb[k + 1] - mb[k]))
    ideal.append(H)
    lo_h, hi_h = min_rows, max(min_rows, int(max_share * H / n))
    out = [0]
    for i in range(1, n):
        b = bounds[i] + damping * (ideal[i] - bounds[i])
        b = int(round(b / align)) * align
        b = max(b, out[-1] + lo_h)                    # not thinner than min_rows ...
        b = min(b, out[-1] + hi_h)                    # ... nor taller than max_share x the mean
        b = min(b, H - (n - i) * lo_h)                # leave room for the bands below
        out.append(b)
    out.append(H)
    for i in range(n - 1, 0, -1):                     # the cap holds for the last bands too: push borders down where a band exceeds it
        if out[i + 1] - out[i] > hi_h:
            out[i] = min(out[i + 1] - lo_h, -(-(out[i + 1] - hi_h) // align) * align)
    return tuple(out)


class _PlaneRef:
    """adapter: objects with a `.p` rfx_plane"""

    def __init__(self, p):
        self.p = p


def _raw_plane(abi, ptr: int, width: int, height: int, pitch: int, fmt: int):
    p = abi.Plane()
    p.ptr, p.width, p.height, p.pitch, p.format = ptr, width, height, pitch, fmt
    return p


def download_band(ctx, stream, downloads, b0: int, b1: int) -> int:
    """rows [b0, b1) of every (rfx_plane, host tensor) pair of `downloads` D2H on `stream`, tightly packed at the start of the host
    tensor (a pair whose tensor is None is skipped); returns the bytes moved"""
    import ctypes as C

    from . import abi

    n = 0
    for plane, out in downloads:
        if out is None:
            continue
        ctx._chk(ctx.lib.rfx_plane_download_rows(ctx.h, stream, C.byref(plane), out.data_ptr(), b0, b1))
        n += (b1 - b0) * plane.width * abi.FMT_BYTES[plane.format]
    return n


def _group_unique_id(ctx, rank, world, unique_id, dist_group):
    """(rank, world, 128-byte NCCL unique id): as given, or from torch.distributed (rank 0 makes the id and broadcasts it)"""
    import ctypes as C

    from . import abi

    if rank is not None and world is not None and unique_id is not None:
        return rank, world, unique_id
    import torch.distributed as dist

    rank, world = dist.get_rank(dist_group), dist.get_world_size(dist_group)
    box = [None]
    if rank == 0:
        buf = C.create_string_buffer(abi.GROUP_ID_BYTES)
        ctx._chk(ctx.lib.rfx_group_get_unique_id(buf))
        box[0] = bytes(buf.raw)
    src = dist.get_global_rank(dist_group, 0) if dist_group is not None else 0
    dist.broadcast_object_list(box, src=src, group=dist_group)
    return rank, world, box[0]


class ShardedSsgiChain:
    """This rank's member of a row-sharded SSGI chain: Python binding of rfx_group_* + rfx_ssgi_chain_render_sharded.

    The 128-byte NCCL unique id travels over torch.distributed (any backend) when a process group is initialised, or is
    passed explicitly (`unique_id`, e.g. read from a file by a host without torch)."""

    # name, bytes/px, sampled anywhere, format
    INPUTS = (("depth", 4, True, "FMT_R32F"), ("gbuffer", 16, False, "FMT_RGBA32F"), ("velocity", 16, True, "FMT_RGBA32F"), ("direct", 8, False, "FMT_RGBA16F"))
    _CHAIN, _ATTACH = "SsgiChain", "rfx_group_attach_chain"  # the member chain's engine class and its collective attach

    def __init__(self, ctx, chain_options, rank: int | None = None, world: int | None = None, unique_id: bytes | None = None,
                 rebalance_every: int = 4, rebalance_lag: int = 2, dist_group=None, traa=None, motion_blur=None):
        """traa: abi.TraaTailOptions (abi.make_traa_tail_options()) to render the TRAA tail too (the same on every rank), or None.
        motion_blur: abi.MotionBlurParams to turn the tail's motion-blur stage on (with traa; set_motion_blur updates it per frame)"""
        import ctypes as C

        from . import abi, engine

        self._abi, self.ctx, self.lib, self._C = abi, ctx, ctx.lib, C
        rank, world, unique_id = _group_unique_id(ctx, rank, world, unique_id, dist_group)
        self.rank, self.world = rank, world
        self.chain = getattr(engine, self._CHAIN)(ctx, chain_options)
        if traa is not None:  # before the attach: the group maps the tail's history plane then
            self.chain.enable_traa(traa)
        if motion_blur is not None:  # before the attach too: the group maps the plane the stage's taps read
            self.chain.set_motion_blur(motion_blur)
        g = C.c_void_p()
        ctx._chk(self.lib.rfx_group_create(ctx.h, unique_id, rank, world, C.byref(g)))
        self.g = g
        ctx._chk(getattr(self.lib, self._ATTACH)(g, self.chain.h))
        ctx._chk(self.lib.rfx_group_set_rebalance(g, int(rebalance_every), int(rebalance_lag)))
        self.rebalance_every = rebalance_every
        self._host = None

    # ---- bands -------------------------------------------------------------------------------------------------------
    @property
    def bounds(self) -> tuple:
        b = (self._C.c_uint32 * (self.world + 1))()
        self.ctx._chk(self.lib.rfx_group_get_bounds(self.g, b))
        return tuple(int(x) for x in b)

    def set_bounds(self, bounds):
        b = (self._C.c_uint32 * (self.world + 1))(*[int(x) for x in bounds])
        self.ctx._chk(self.lib.rfx_group_set_bounds(self.g, b))

    @property
    def band(self) -> tuple:
        b = self.bounds
        return b[self.rank], b[self.rank + 1]

    @property
    def uses_peer_reads(self) -> bool:
        """True: history rows are read in place on their owner over NVLink; False: replicated by an NCCL exchange every frame (fallback)"""
        return bool(self.lib.rfx_group_uses_peer_reads(self.g))

    @property
    def last_costs(self) -> list:
        c = (self._C.c_float * self.world)()
        self.ctx._chk(self.lib.rfx_group_last_costs(self.g, c))
        return [float(x) for x in c]

    def begin_frame(self) -> tuple:
        """Collective in lockstep (no communication): applies the cost-driven border move that is due for the next frame and
        returns the borders that frame will use.  render() calls it implicitly; the host path calls it before its uploads."""
        b = (self._C.c_uint32 * (self.world + 1))()
        self.ctx._chk(self.lib.rfx_group_begin_frame(self.g, b))
        return tuple(int(x) for x in b)

    # ---- device-resident frame ---------------------------------------------------------------------------------------
    def set_motion_blur(self, params):
        """this frame's MotionBlurEffect uniforms (the same on every rank; the stage was turned on at construction)"""
        self.chain.set_motion_blur(params)

    def set_effects(self, params):
        """the cosmetic stage (engine.SsgiChain.set_effects) with this frame's values, or None to turn it off; the same on every rank, any
        frame (the stage keeps no plane the group maps)"""
        self.chain.set_effects(params)

    def set_compose(self, params):
        """the compose stage (engine.SsgiChain.set_compose: output 9, K5 over output 0), or None to turn it off; the same on every rank,
        any frame (it runs on the band and keeps no plane the group maps)"""
        self.chain.set_compose(params)

    def render(self, cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved: bool, stream=None):
        """Collective: one frame from full-frame device planes; this rank renders its band and joins the frame's collectives.  Both
        phases of a frame with the motion-blur stage (render_sharded, then render_sharded_finish; the latter is a no-op otherwise)."""
        f = self.chain._frame(cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved)
        self.ctx._chk(self.lib.rfx_ssgi_chain_render_sharded(self.chain.h, stream, self._C.byref(f)))
        self._finish(stream)

    def _finish(self, stream):
        fn = "rfx_ao_chain_render_sharded_finish" if self._CHAIN == "AoChain" else "rfx_ssgi_chain_render_sharded_finish"
        self.ctx._chk(getattr(self.lib, fn)(self.chain.h, stream))

    def download_band(self, which: int | None = None):
        """this rank's rows of chain output `which` (default: the chain's) of the last frame (numpy)"""
        b0, b1 = self.band_of_last_frame
        return self.chain.download(which)[b0:b1]

    @property
    def band_of_last_frame(self) -> tuple:
        b = (self._C.c_uint32 * (self.world + 1))()
        self.ctx._chk(self.lib.rfx_group_get_last_bounds(self.g, b))
        return int(b[self.rank]), int(b[self.rank + 1])

    def finish(self):
        self.ctx.sync()

    # ---- host-buffer path --------------------------------------------------------------------------------------------
    # Every rank holds (or maps) the frame's host planes but moves only its share over PCIe: its own rows of depth and velocity —
    # the two input planes sampled anywhere on screen (ray-march taps, reprojected uv), which are then completed from the other
    # ranks' uploads with one NCCL exchange over NVLink (rfx_group_allgather_rows: the path's one real input exchange) — and the
    # K1-range rows (+1) of the G-buffer and the direct light.  H2D, kernels and D2H run on three streams with two staging sets,
    # like rfx_ssgi_chain_submit_host on one GPU.
    MAX_SHARE = 4.0

    def _host_init(self):
        import torch

        abi = self._abi
        dev = torch.device("cuda", self.ctx.device)
        W, H = self.chain.opt.width, self.chain.opt.height
        h = dict(torch=torch, W=W, H=H, staging=[], frames=0)
        for _ in range(2):
            st = {}
            for name, bpp, _g, fmt in self.INPUTS:
                t = torch.zeros(H * W * bpp, dtype=torch.uint8, device=dev)
                st[name] = (t, _raw_plane(abi, t.data_ptr(), W, H, W * bpp, getattr(abi, fmt)), W * bpp)
            h["staging"].append(st)
        h["up"], h["dn"] = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        h["main"] = torch.cuda.ExternalStream(self.ctx.stream, device=dev)
        h["ev_up"] = [torch.cuda.Event() for _ in range(2)]
        h["ev_rendered"] = [torch.cuda.Event() for _ in range(2)]
        h["ev_dn"] = [torch.cuda.Event() for _ in range(2)]
        h["bytes"] = (0, 0)
        self._host = h

    def submit_host(self, cam, host: dict, camera_pos, camera_moved: bool, out_host, out_color=None):
        """One frame from host planes (dict name -> CPU tensor of the FULL frame, pinned for asynchronous copies) to this rank's
        rows of `composed`, written to the start of out_host (CPU float32 tensor of at least MAX_SHARE x the mean band height x W x 4),
        and of the compose stage's image (output 9, set_compose first), written to the start of out_color (CPU float16 tensor of the
        same number of texels).  Either may be None, not both.  Returns the band (row0, row1) the rows belong to, after enqueueing.  Not
        with the TRAA tail: the rows uploaded here (local_input_rows) are sized for the chain without it."""
        abi = self._abi
        if self.chain.traa is not None:
            raise abi.RfxError(f"rfx status {abi.ERR_UNSUPPORTED}: submit_host: the sharded host path does not render the TRAA tail")
        o = self.chain.opt
        if o.mode != abi.MODE_SSGI or o.denoise_mode != 0:
            raise abi.RfxError(f"rfx status {abi.ERR_UNSUPPORTED}: submit_host: the sharded host path renders the fast SSGI chain only "
                               "(mode SSGI, denoiseMode \"full\"): its upload rows are planned for that chain")
        if out_host is None and out_color is None:
            raise abi.RfxError(f"rfx status {abi.ERR_INVALID_ARG}: submit_host: out_host and out_color are both None")
        if out_color is not None and self.chain.compose is None:
            raise abi.RfxError(f"rfx status {abi.ERR_NOT_READY}: submit_host: out_color is the compose stage's image, and the stage is off")

        def rows(bounds):
            return ShardPlan(o.height, self.world, self.rank, 2 * o.denoise_iterations, o.radius, True, bounds=bounds, width=o.width).local_input_rows

        def render(st, plane):
            self.render(cam, plane("depth"), plane("gbuffer"), plane("velocity"), plane("direct"), camera_pos, camera_moved)
            # `composed` and the compose stage's image are double-buffered by frame parity: the planes of frame i are next written by
            # frame i+2, which waits for this frame's D2H through ev_dn, so the rows go D2H straight from the planes
            return [(self.chain.output(0), out_host), (self.chain.output(9) if out_color is not None else None, out_color)]

        return self._submit_host_frame(host, rows, render)

    def _submit_host_frame(self, host: dict, local_rows, render):
        """submit_host's pipeline: this rank's uploads into staging set (frame & 1) on the copy stream, the all-gather of the planes sampled
        anywhere, render(staging set, plane of name) -> the (plane, host tensor) pairs whose band goes D2H, then those bands on the third
        stream (download_band).  local_rows(bounds): the rows of the per-pixel input planes this rank reads."""
        if self._host is None:
            self._host_init()
        h = self._host
        torch, W, H = h["torch"], h["W"], h["H"]
        bounds = self.begin_frame()
        b0, b1 = bounds[self.rank], bounds[self.rank + 1]
        l0, l1 = local_rows(bounds)
        k = h["frames"] & 1
        st = h["staging"][k]
        h2d = 0
        with torch.cuda.stream(h["up"]):
            if h["frames"] >= 2:
                h["up"].wait_event(h["ev_rendered"][k])   # frame i-2 no longer reads this staging set
            for name, bpp, anywhere, _fmt in self.INPUTS:
                if host.get(name) is None:
                    continue
                t, _pl, pitch = st[name]
                a, b = ((b0, b1) if anywhere else (l0, l1)) if self.world > 1 else (0, H)
                t.view(H, pitch)[a:b].copy_(host[name].view(torch.uint8).view(H, pitch)[a:b], non_blocking=True)
                h2d += (b - a) * pitch
            h["ev_up"][k].record(h["up"])
        with torch.cuda.stream(h["main"]):
            h["main"].wait_event(h["ev_up"][k])
            if h["frames"] >= 2:
                h["main"].wait_event(h["ev_dn"][k])       # what frame i-2's D2H read (the set's staged output) may be written again
        if self.world > 1:  # complete the planes sampled anywhere from the other ranks' uploads (NVLink), ordered on the context stream
            bnd = (self._C.c_uint32 * (self.world + 1))(*bounds)
            for name, _bpp, anywhere, _fmt in self.INPUTS:
                if anywhere and host.get(name) is not None:
                    self.ctx._chk(self.lib.rfx_group_allgather_rows(self.g, None, self._C.byref(st[name][1]), bnd))
        downloads = render(st, lambda n: _PlaneRef(st[n][1]) if host.get(n) is not None else None)
        with torch.cuda.stream(h["main"]):
            h["ev_rendered"][k].record(h["main"])
        with torch.cuda.stream(h["dn"]):
            h["dn"].wait_event(h["ev_rendered"][k])
            nbytes = download_band(self.ctx, h["dn"].cuda_stream, downloads, b0, b1)
            h["ev_dn"][k].record(h["dn"])
        h["frames"] += 1
        h["bytes"] = (h2d, nbytes)
        return b0, b1

    def wait_host(self, max_in_flight: int = 0):
        h = self._host
        if not h or h["frames"] == 0:
            return
        n = h["frames"]
        if max_in_flight <= 0:
            h["ev_dn"][(n - 1) & 1].synchronize()
        elif n >= 2:
            h["ev_dn"][(n - 2) & 1].synchronize()

    @property
    def host_bytes_per_frame(self):
        """(H2D, D2H) bytes this rank moved for the last submitted frame"""
        return self._host["bytes"] if self._host else (0, 0)

    def close(self):
        self.ctx.sync()
        if self.g:
            self.lib.rfx_group_destroy(self.g)
            self.g = None
        self.chain.close()


class InProcessGroup:
    """`world` members of a row-sharded group inside ONE process (rfx_group_create_inprocess / rfx_group_attach_chains_inprocess): every member
    owns a chain (any options a group takes: fast_math on, resolution_scale 1) and a band; the members read each other's history planes through plain device pointers.  With one context this
    renders the bands one after the other on one GPU — the N-band logic (halo recomputation, owner lookup of history rows, carried texels,
    moving borders) without N GPUs; with one context per device it is a single-process multi-GPU host."""

    _CHAIN, _ATTACH = "SsgiChain", "rfx_group_attach_chains_inprocess"  # the members' engine class and their attach

    def __init__(self, ctxs, chain_options, world: int, traa=None, motion_blur=None):
        """traa: abi.TraaTailOptions to render the TRAA tail on every member, or None; motion_blur: abi.MotionBlurParams to turn the tail's
        motion-blur stage on (set_motion_blur updates it per frame)"""
        import ctypes as C

        from . import abi, engine

        self._C, self.world = C, world
        self.ctxs = list(ctxs) if isinstance(ctxs, (list, tuple)) else [ctxs] * world
        assert len(self.ctxs) == world
        self.lib = self.ctxs[0].lib
        self.chains = [getattr(engine, self._CHAIN)(c, chain_options) for c in self.ctxs]
        if traa is not None:
            for ch in self.chains:
                ch.enable_traa(traa)
        if motion_blur is not None:
            for ch in self.chains:
                ch.set_motion_blur(motion_blur)
        self.groups = []
        for r, c in enumerate(self.ctxs):
            g = C.c_void_p()
            c._chk(self.lib.rfx_group_create_inprocess(c.h, r, world, C.byref(g)))
            self.groups.append(g)
        ga = (C.c_void_p * world)(*[g.value for g in self.groups])
        ca = (C.c_void_p * world)(*[ch.h.value if hasattr(ch.h, "value") else ch.h for ch in self.chains])
        self.ctxs[0]._chk(getattr(self.lib, self._ATTACH)(ga, ca, world))

    @property
    def bounds(self) -> tuple:
        b = (self._C.c_uint32 * (self.world + 1))()
        self.ctxs[0]._chk(self.lib.rfx_group_get_bounds(self.groups[0], b))
        return tuple(int(x) for x in b)

    def set_bounds(self, bounds):
        """new borders for the next frame (every member gets the same ones)"""
        b = (self._C.c_uint32 * (self.world + 1))(*[int(x) for x in bounds])
        for c, g in zip(self.ctxs, self.groups):
            c._chk(self.lib.rfx_group_set_bounds(g, b))

    def set_motion_blur(self, params):
        """this frame's MotionBlurEffect uniforms for every member (the stage was turned on at construction)"""
        for ch in self.chains:
            ch.set_motion_blur(params)

    def set_effects(self, params):
        """the cosmetic stage with this frame's values for every member, or None to turn it off (any frame)"""
        for ch in self.chains:
            ch.set_effects(params)

    def set_compose(self, params):
        """the compose stage (output 9) for every member, or None to turn it off (any frame)"""
        for ch in self.chains:
            ch.set_compose(params)

    def render(self, cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved: bool, wait: bool = True):
        """one frame: every member renders its band; all of them finish before the next frame starts (the host is the barrier).
        wait=False skips the host wait: only for members that share one context, whose stream orders the members and the frames."""
        self._last_bounds = self.bounds
        for c, ch in zip(self.ctxs, self.chains):
            f = ch._frame(cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved)
            c._chk(self.lib.rfx_ssgi_chain_render_sharded(ch.h, None, self._C.byref(f)))
        self._finish(wait)

    def _finish(self, wait: bool):
        """phase 2 of every member (a no-op without the motion-blur stage), after phase 1 of every member: one stream orders them; members
        on several contexts are synchronised in between"""
        fn = "rfx_ao_chain_render_sharded_finish" if self._CHAIN == "AoChain" else "rfx_ssgi_chain_render_sharded_finish"
        several = len(set(self.ctxs)) > 1
        if several:
            for c in set(self.ctxs):
                c.sync()
        for c, ch in zip(self.ctxs, self.chains):
            c._chk(getattr(self.lib, fn)(ch.h, None))
        if wait or several:
            for c in set(self.ctxs):
                c.sync()

    def download(self, which: int = 0):
        """output `which` of the last frame, assembled from the members' bands"""
        import numpy as np

        b = self._last_bounds
        return np.concatenate([ch.download(which)[b[r]:b[r + 1]] for r, ch in enumerate(self.chains)], axis=0)

    def close(self):
        for c, g in zip(self.ctxs, self.groups):
            c.sync()
            self.lib.rfx_group_destroy(g)
        for ch in self.chains:
            ch.close()


def _render_ao_band(ctx, chain, stream, frame: tuple, traa_cam, camera_moved: bool):
    """rfx_ao_chain_render_sharded (traa_cam None) or rfx_ao_chain_render_sharded_traa for one member; frame: AoChain._frame's arguments"""
    import ctypes as C

    f = chain._frame(*frame)
    if traa_cam is None:
        ctx._chk(ctx.lib.rfx_ao_chain_render_sharded(chain.h, stream, C.byref(f)))
    else:
        t = chain._traa_frame(traa_cam, camera_moved)
        ctx._chk(ctx.lib.rfx_ao_chain_render_sharded_traa(chain.h, stream, C.byref(f), C.byref(t)))


class _CudaRows:
    """rows [0, n) x `row_bytes` bytes of device memory at `ptr` with a row pitch, for torch.as_tensor (__cuda_array_interface__)"""

    def __init__(self, ptr: int, n: int, row_bytes: int, pitch: int):
        self.__cuda_array_interface__ = {"shape": (n, row_bytes), "strides": (pitch, 1), "typestr": "|u1", "data": (ptr, False), "version": 2}


class ShardedAoChain(ShardedSsgiChain):
    """This rank's member of a row-sharded AO chain: rfx_group_* + rfx_ao_chain_render_sharded.  The constructor (chain_options:
    engine.ao_chain_options(...)), bands, rebalancing and the unique-id exchange are ShardedSsgiChain's.

    Host-buffer path (submit_host / wait_host, without the TRAA tail): every rank moves only its share over PCIe.  depth, which K6 / K6h
    sample anywhere, goes up as the rank's band and is completed from the other ranks' bands with rfx_group_allgather_rows; velocity,
    the normal plane and the scene colour go up as AoShardPlan.local_input_rows.  The rank's band of the K7 output (or, without a scene
    colour, of output 1) comes back D2H.  H2D, kernels and D2H run on three streams with two staging sets, as
    rfx_ao_chain_submit_host does on one GPU."""

    _CHAIN, _ATTACH = "AoChain", "rfx_group_attach_ao_chain"
    INPUTS = (("depth", 4, True, "FMT_R32F"), ("velocity", 16, False, "FMT_RGBA32F"), ("normal", 4, False, "FMT_RGBA8"), ("input", 8, False, "FMT_RGBA16F"))

    def render(self, cam_u, depth, velocity, normal=None, inp=None, out=None, stream=None, traa_cam=None, camera_moved: bool = True):
        """Collective: one frame from full-frame device planes; this rank renders its band and joins the frame's collective.
        traa_cam / camera_moved: as AoChain.render, with the TRAA tail on."""
        _render_ao_band(self.ctx, self.chain, stream, (cam_u, depth, velocity, normal, inp, out), traa_cam, camera_moved)
        self._finish(stream)

    def _host_init(self):
        super()._host_init()
        h, abi = self._host, self._abi
        W, H = h["W"], h["H"]
        for st in h["staging"]:  # the plane the set's D2H reads: K7's output, or the band of output 1 copied out of the chain's plane
            t = h["torch"].zeros(H * W * 8, dtype=h["torch"].uint8, device=st["depth"][0].device)
            st["out"] = (t, _raw_plane(abi, t.data_ptr(), W, H, W * 8, abi.FMT_RGBA16F), W * 8)

    def submit_host(self, cam_u: dict, host: dict, out_host):
        """One frame from host planes (dict name -> CPU tensor of the FULL frame, pinned for asynchronous copies: depth, velocity, and
        normal with use_normal_plane, input for K7) to this rank's rows of the K7 output (with `input`) or of output 1 (without), written to
        the start of out_host (CPU tensor of at least MAX_SHARE x the mean band height x W x 8 bytes).  Returns the band (row0, row1) the
        rows belong to, after enqueueing.  Not with the TRAA tail (ERR_UNSUPPORTED): its pass reads velocity at reprojected uvs, which the
        uploaded rows (AoShardPlan.local_input_rows) do not cover."""
        abi = self._abi
        if self.chain.traa is not None:
            raise abi.RfxError(f"rfx status {abi.ERR_UNSUPPORTED}: submit_host: the sharded host path does not render the TRAA tail")
        if host.get("depth") is None or host.get("velocity") is None:
            raise abi.RfxError("submit_host: depth and velocity are required")
        o = self.chain.opt

        def rows(bounds):
            return AoShardPlan(o.width, o.height, (bounds[self.rank], bounds[self.rank + 1]), o.iterations, o.radius).local_input_rows

        def render(st, plane):
            out = st["out"]
            with_k7 = host.get("input") is not None
            self.render(cam_u, plane("depth"), plane("velocity"), plane("normal"), plane("input"), _PlaneRef(out[1]) if with_k7 else None)
            if not with_k7:
                # output 1 is rendered in place (alone) or by frame parity (in a group), and the next frame's kernels may write it while
                # this band is still going D2H: copy the band into the set's plane on the context stream first
                torch, (b0, b1) = self._host["torch"], self.band_of_last_frame
                p = self.chain.output(1)
                src = torch.as_tensor(_CudaRows(p.ptr + b0 * p.pitch, b1 - b0, p.width * 8, p.pitch), device=out[0].device)
                with torch.cuda.stream(self._host["main"]):
                    out[0].view(self._host["H"], out[2])[b0:b1].copy_(src)
            return [(out[1], out_host)]

        return self._submit_host_frame(host, rows, render)


class InProcessAoGroup(InProcessGroup):
    """InProcessGroup for the AO chain (rfx_group_attach_ao_chains_inprocess): every member owns an AoChain with the same options
    (chain_options: engine.ao_chain_options(...))."""

    _CHAIN, _ATTACH = "AoChain", "rfx_group_attach_ao_chains_inprocess"

    def render(self, cam_u, depth, velocity, normal=None, inp=None, out=None, wait: bool = True, traa_cam=None, camera_moved: bool = True):
        """one frame: every member renders its band (its rows of `out` too); all of them finish before the next frame starts.
        traa_cam / camera_moved: as AoChain.render, with the TRAA tail on."""
        self._last_bounds = self.bounds
        for c, ch in zip(self.ctxs, self.chains):
            _render_ao_band(c, ch, None, (cam_u, depth, velocity, normal, inp, out), traa_cam, camera_moved)
        self._finish(wait)
