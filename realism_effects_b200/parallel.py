"""Row-band sharding of the SSGI chain and the AO chain across N GPUs (one process per GPU).

The product path is native: `rfx_group_*` / `rfx_ssgi_chain_render_sharded` in csrc/rfx_group.inl (C ABI, include/rfx.h).
This module is the Python host binding of that API (`ShardedSsgiChain`) plus a pure-Python mirror of its host arithmetic
(`ShardPlan`, `rebalance`) that the CPU tests check against the exported C functions `rfx_shard_ranges` / `rfx_shard_rebalance`
and drive with the oracle as compute (tests/test_sharding_cpu.py).

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

Adaptive bands: one contiguous band per rank; every few frames the borders move towards equal device-timed cost
(`rfx_shard_rebalance`: cost per row piecewise constant over the measured bands, damped, 16-row aligned; every rank derives the
same borders from the same gathered times).  All cross-frame state lives in the peer-readable planes, so borders move freely
between frames and the result stays bit-identical to the single-GPU chain (tests/test_gpu_multi.py).
"""
from __future__ import annotations

import math
from dataclasses import dataclass


@dataclass
class ShardPlan:
    """Row ranges [a, b) per launch of one frame, in chain order: K1, K2, K3 pass 0..n-1, K4,
    for every row block this rank owns."""

    height: int
    world: int
    rank: int
    n_poisson_passes: int  # 2 * denoiseIterations
    radius: float
    ssgi_mode: bool = True
    blocks_per_rank: int = 1
    mirror: bool = False  # True: odd super-blocks are assigned in REVERSE rank order (boustrophedon), see block_of()
    bounds: tuple | None = None  # explicit band borders (world + 1 ascending rows, 0 .. height): one contiguous band per rank
    width: int | None = None     # frame width: portrait frames (H > W) stretch the Poisson taps' row reach by H / W
    traa: bool = False           # the TRAA tail runs as one more launch after K4 (rfx_ssgi_chain_enable_traa)
    denoise_mode: int = 0        # 0 "full"; 1 "full_temporal" / 2 "temporal" run no Poisson pass, so their ranges are those of 0 passes

    K2_NEIGHBOURHOOD_ROWS = 2  # 5x5 clamp window (reproject.frag:57-59)
    K4_INPUT_ROWS = 1          # literal bilinear fetch of the LINEAR Poisson targets at the pixel centre
    # `composed` rows the TRAA tail reads around its band (include/rfx.h RFX_TRAA_TAIL_ROWS): 2 for the TRAA clamp window, 1 because
    # those taps are LINEAR fetches at texel centres (the reason of K4_INPUT_ROWS), 1 for K9's LINEAR fetch of the accumulated plane at
    # the pixel centre; the TRAA form takes no derivative, so no quad row
    TRAA_TAIL_ROWS = 4

    def block_of(self, rank: int, j: int):
        """rows of the block `rank` owns inside super-block j.  With `mirror`, odd super-blocks run in reverse rank order, so a
        rank that gets the cheapest end of one super-block (sky) gets the most expensive end of the next (floor): 2 blocks per
        rank already balance a vertical cost gradient, at half the halo recompute of a 4-block cyclic assignment."""
        if self.bounds is not None:
            return (self.bounds[rank], self.bounds[rank + 1])
        pos = (self.world - 1 - rank) if (self.mirror and j % 2 == 1) else rank
        b = j * self.world + pos
        return (b * self.block_rows, (b + 1) * self.block_rows)

    def reversed_order(self, j: int) -> bool:
        return self.mirror and j % 2 == 1

    @property
    def p2p(self) -> bool:
        """the exchange cannot be a rank-ordered in-place all-gather (mirrored order or unequal bands)"""
        return self.mirror or self.bounds is not None

    def __post_init__(self):
        if self.bounds is not None:
            b = tuple(int(x) for x in self.bounds)
            if len(b) != self.world + 1 or b[0] != 0 or b[-1] != self.height or any(b[i] >= b[i + 1] for i in range(self.world)):
                raise ValueError(f"bounds {b} are not {self.world + 1} ascending rows from 0 to {self.height}")
            self.bounds, self.blocks_per_rank, self.block_rows = b, 1, None
            self.blocks = [self.block_of(self.rank, 0)]
            self.rows_per_rank = self.blocks[0][1] - self.blocks[0][0]
            self.r0, self.r1 = self.blocks[0]
            self.poisson_halo = self._halo()
            return
        nb = self.world * self.blocks_per_rank
        if self.height % nb:
            raise ValueError(f"height {self.height} is not divisible by world size x blocks per rank = {nb}")
        self.block_rows = self.height // nb
        self.rows_per_rank = self.block_rows * self.blocks_per_rank
        self.blocks = [self.block_of(self.rank, j) for j in range(self.blocks_per_rank)]
        self.r0, self.r1 = self.blocks[0]  # (single-block plans: the contiguous band)
        self.poisson_halo = self._halo()

    def _halo(self) -> int:
        """rows a Poisson tap can reach: the offset is rotated after the division by the resolution (poisson_denoise.frag:183-189),
        so the row reach is radius * max(1, H / W); + 1 for the bilinear footprint / the quad-derivative helper row"""
        stretch = max(1.0, self.height / self.width) if self.width else 1.0
        return int(math.ceil(self.radius * stretch)) + 1

    def _expand(self, rng, rows):
        return (max(0, rng[0] - rows), min(self.height, rng[1] + rows))

    @property
    def passes(self) -> int:
        """Poisson passes the ranges are planned for: n_poisson_passes in denoiseMode "full", else none (Denoiser.js:47-52).  The native
        chain maps a full_temporal / temporal frame's K1, K2, K4 (and tail) launches onto these ranges (rfx_ssgi_chain_render_sharded)."""
        return self.n_poisson_passes if self.denoise_mode == 0 else 0

    def ranges_for(self, own) -> list:
        n = self.passes
        k4 = self._expand(own, self.TRAA_TAIL_ROWS) if self.traa else own
        k3 = [None] * n
        nxt = k4
        if n:
            k3[n - 1] = self._expand(k4, self.K4_INPUT_ROWS)
            for j in range(n - 2, -1, -1):
                k3[j] = self._expand(k3[j + 1], self.poisson_halo)
            nxt = self._expand(k3[0], self.poisson_halo)
        k2 = nxt
        k1 = self._expand(k2, self.K2_NEIGHBOURHOOD_ROWS)
        return [k1, k2, *k3, k4] + ([own] if self.traa else [])  # K4 runs in both modes (SSR composes with inputType specular)

    @property
    def ranges(self) -> list:
        """single-block plans: the per-launch ranges of the band"""
        return self.ranges_for(self.blocks[0])

    @property
    def block_ranges(self) -> list:
        """[block][launch] -> (row0, row1)"""
        return [self.ranges_for(b) for b in self.blocks]

    @property
    def n_launches(self) -> int:
        return 3 + self.passes + (1 if self.traa else 0)

    def super_block(self, j: int):
        """rows of super-block j: N consecutive blocks, one per rank, in rank order (an in-place all-gather unit)"""
        return (j * self.world * self.block_rows, (j + 1) * self.world * self.block_rows)

    @property
    def recompute_overhead(self) -> float:
        """extra rows launched / rows owned (the price of exchanging nothing per pass)"""
        tot = sum((b - a) for rs in self.block_ranges for a, b in rs)
        return tot / (self.n_launches * self.rows_per_rank) - 1.0

    @property
    def local_input_rows(self) -> list:
        """Rows of the PER-PIXEL input planes (G-buffer, direct light) this rank reads: the K1 range of each block (it contains
        every later launch's range and the rows its Poisson taps reach) + 1 row each side, because K1's literal bilinear fetch
        of the direct-light plane at the pixel centre touches row y +- 1 whenever ((y + .5) / H) * H - .5 is not exactly y.
        The planes sampled at arbitrary screen positions (depth: ray-march taps; velocity: reprojected uv) are needed whole."""
        return [self._expand(rs[0], 1) for rs in self.block_ranges]

    @property
    def gathered_planes(self):
        """chain outputs (`rfx_ssgi_chain_output` index) that are all-gathered after the frame; `composed` first"""
        return (0, 4, 5) if self.ssgi_mode else (4,)


@dataclass
class AoShardPlan:
    """Row ranges [a, b) per launch of one AO chain frame for the band `own`, in chain order: K6 / K6h, K3 pass 0..2*iterations-1, K7
    (mirror of rfx_ao_shard_ranges).  No AO pass reads a produced plane at an arbitrary uv, so the only cross-row reads are K7's LINEAR
    fetch at the pixel centre (1 row) and the Poisson taps (the halo of ShardPlan)."""

    width: int
    height: int
    own: tuple
    iterations: int
    radius: float

    K7_INPUT_ROWS = 1

    @property
    def poisson_halo(self) -> int:
        return int(math.ceil(abs(self.radius) * max(1.0, self.height / self.width))) + 1

    @property
    def n_launches(self) -> int:
        return 2 + 2 * self.iterations

    @property
    def ranges(self) -> list:
        expand = lambda r, rows: (max(0, r[0] - rows), min(self.height, r[1] + rows))  # noqa: E731
        out = [tuple(self.own)]
        r = expand(out[0], self.K7_INPUT_ROWS)
        for _ in range(2 * self.iterations):
            out.append(r)
            r = expand(r, self.poisson_halo)
        out.append(r)
        return out[::-1]


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

    INPUTS = (("depth", 4, True), ("gbuffer", 16, False), ("velocity", 16, True), ("direct", 8, False))  # name, bytes/px, sampled anywhere

    def __init__(self, ctx, chain_options, rank: int | None = None, world: int | None = None, unique_id: bytes | None = None,
                 rebalance_every: int = 4, rebalance_lag: int = 2, dist_group=None, traa=None):
        """traa: abi.TraaTailOptions (abi.make_traa_tail_options()) to render the TRAA tail too (the same on every rank), or None"""
        import ctypes as C

        from . import abi, engine

        self._abi, self.ctx, self.lib, self._C = abi, ctx, ctx.lib, C
        rank, world, unique_id = _group_unique_id(ctx, rank, world, unique_id, dist_group)
        self.rank, self.world = rank, world
        self.chain = engine.SsgiChain(ctx, chain_options)
        if traa is not None:  # before the attach: the group maps the tail's history plane then
            self.chain.enable_traa(traa)
        g = C.c_void_p()
        ctx._chk(self.lib.rfx_group_create(ctx.h, unique_id, rank, world, C.byref(g)))
        self.g = g
        ctx._chk(self.lib.rfx_group_attach_chain(g, self.chain.h))
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
    def render(self, cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved: bool, stream=None):
        """Collective: one frame from full-frame device planes; this rank renders its band and joins the frame's collective."""
        f = self.chain._frame(cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved)
        self.ctx._chk(self.lib.rfx_ssgi_chain_render_sharded(self.chain.h, stream, self._C.byref(f)))

    def download_band(self, which: int = 0):
        """this rank's rows of chain output `which` of the last frame (numpy)"""
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
        fmts = dict(depth=abi.FMT_R32F, gbuffer=abi.FMT_RGBA32F, velocity=abi.FMT_RGBA32F, direct=abi.FMT_RGBA16F)
        h = dict(torch=torch, W=W, H=H, staging=[], frames=0)
        for _ in range(2):
            st = {}
            for name, bpp, _g in self.INPUTS:
                t = torch.zeros(H * W * bpp, dtype=torch.uint8, device=dev)
                st[name] = (t, _raw_plane(abi, t.data_ptr(), W, H, W * bpp, fmts[name]), W * bpp)
            h["staging"].append(st)
        cap = H if self.world == 1 else min(H, int(self.MAX_SHARE * H / self.world) + 16)
        h["out_dev"] = [torch.empty(cap * W * 16, dtype=torch.uint8, device=dev) for _ in range(2)]
        h["up"], h["dn"] = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        h["main"] = torch.cuda.ExternalStream(self.ctx.stream, device=dev)
        h["ev_up"] = [torch.cuda.Event() for _ in range(2)]
        h["ev_rendered"] = [torch.cuda.Event() for _ in range(2)]
        h["ev_dn"] = [torch.cuda.Event() for _ in range(2)]
        h["bytes"] = (0, 0)
        self._host = h

    def submit_host(self, cam, host: dict, camera_pos, camera_moved: bool, out_host):
        """One frame from host planes (dict name -> CPU tensor of the FULL frame, pinned for asynchronous copies) to this rank's
        rows of `composed`, written to the start of out_host (CPU float32 tensor of at least MAX_SHARE x the mean band height).
        Returns the band (row0, row1) the rows belong to, after enqueueing.  Not with the TRAA tail: the rows uploaded here
        (local_input_rows) are sized for the chain without it."""
        if self.chain.traa is not None:
            raise self._abi.RfxError(f"rfx status {self._abi.ERR_UNSUPPORTED}: submit_host: the sharded host path does not render the TRAA tail")
        o = self.chain.opt
        if o.mode != self._abi.MODE_SSGI or o.denoise_mode != 0:
            raise self._abi.RfxError(f"rfx status {self._abi.ERR_UNSUPPORTED}: submit_host: the sharded host path renders the fast SSGI chain only "
                                     "(mode SSGI, denoiseMode \"full\"): its upload rows are planned for that chain")
        if self._host is None:
            self._host_init()
        h = self._host
        torch, W, H = h["torch"], h["W"], h["H"]
        bounds = self.begin_frame()
        b0, b1 = bounds[self.rank], bounds[self.rank + 1]
        plan = ShardPlan(H, self.world, self.rank, 2 * self.chain.opt.denoise_iterations, self.chain.opt.radius, True, bounds=bounds, width=W)
        l0, l1 = plan.local_input_rows[0]
        k = h["frames"] & 1
        st = h["staging"][k]
        h2d = 0
        with torch.cuda.stream(h["up"]):
            if h["frames"] >= 2:
                h["up"].wait_event(h["ev_rendered"][k])   # frame i-2 no longer reads this staging set
            for name, bpp, anywhere in self.INPUTS:
                if host.get(name) is None:
                    continue
                t, _pl, pitch = st[name]
                a, b = ((b0, b1) if anywhere else (l0, l1)) if self.world > 1 else (0, H)
                t.view(H, pitch)[a:b].copy_(host[name].view(torch.uint8).view(H, pitch)[a:b], non_blocking=True)
                h2d += (b - a) * pitch
            h["ev_up"][k].record(h["up"])
        with torch.cuda.stream(h["main"]):
            h["main"].wait_event(h["ev_up"][k])
        if self.world > 1:  # complete depth / velocity from the other ranks' uploads (NVLink), ordered on the context stream
            bnd = (self._C.c_uint32 * (self.world + 1))(*bounds)
            for name, _bpp, anywhere in self.INPUTS:
                if anywhere and host.get(name) is not None:
                    self.ctx._chk(self.lib.rfx_group_allgather_rows(self.g, None, self._C.byref(st[name][1]), bnd))
        pw = lambda n: _PlaneRef(st[n][1]) if host.get(n) is not None else None  # noqa: E731
        self.render(cam, pw("depth"), pw("gbuffer"), pw("velocity"), pw("direct"), camera_pos, camera_moved)
        p = self.chain.output(0)
        nbytes = (b1 - b0) * W * 16
        with torch.cuda.stream(h["main"]):
            h["ev_rendered"][k].record(h["main"])
        with torch.cuda.stream(h["dn"]):
            h["dn"].wait_event(h["ev_rendered"][k])
            # `composed` is double-buffered by frame parity: the plane of frame i is next written by frame i+2, which waits for this
            # copy through ev_dn (wait_host is called with at most one frame in flight), so the rows go D2H straight from the plane
            self.ctx._chk(self.lib.rfx_plane_download_rows(self.ctx.h, h["dn"].cuda_stream, self._C.byref(p), out_host.data_ptr(), b0, b1))
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

    def __init__(self, ctxs, chain_options, world: int, traa=None):
        """traa: abi.TraaTailOptions to render the TRAA tail on every member, or None"""
        import ctypes as C

        from . import abi, engine

        self._C, self.world = C, world
        self.ctxs = list(ctxs) if isinstance(ctxs, (list, tuple)) else [ctxs] * world
        assert len(self.ctxs) == world
        self.lib = self.ctxs[0].lib
        self.chains = [engine.SsgiChain(c, chain_options) for c in self.ctxs]
        if traa is not None:
            for ch in self.chains:
                ch.enable_traa(traa)
        self.groups = []
        for r, c in enumerate(self.ctxs):
            g = C.c_void_p()
            c._chk(self.lib.rfx_group_create_inprocess(c.h, r, world, C.byref(g)))
            self.groups.append(g)
        ga = (C.c_void_p * world)(*[g.value for g in self.groups])
        ca = (C.c_void_p * world)(*[ch.h.value if hasattr(ch.h, "value") else ch.h for ch in self.chains])
        self.ctxs[0]._chk(self.lib.rfx_group_attach_chains_inprocess(ga, ca, world))

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

    def render(self, cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved: bool, wait: bool = True):
        """one frame: every member renders its band; all of them finish before the next frame starts (the host is the barrier).
        wait=False skips the host wait: only for members that share one context, whose stream orders the members and the frames."""
        self._last_bounds = self.bounds
        for c, ch in zip(self.ctxs, self.chains):
            f = ch._frame(cam, depth, gbuffer, velocity, direct_light, camera_pos, camera_moved)
            c._chk(self.lib.rfx_ssgi_chain_render_sharded(ch.h, None, self._C.byref(f)))
        if wait or len(set(self.ctxs)) > 1:
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


class ShardedAoChain(ShardedSsgiChain):
    """This rank's member of a row-sharded AO chain: rfx_group_* + rfx_ao_chain_render_sharded.  Bands, rebalancing and the unique-id
    exchange are ShardedSsgiChain's; the host-buffer path is not (out of scope for AO)."""

    def __init__(self, ctx, ao_options, rank: int | None = None, world: int | None = None, unique_id: bytes | None = None,
                 rebalance_every: int = 4, rebalance_lag: int = 2, dist_group=None):
        import ctypes as C

        from . import abi, engine

        self._abi, self.ctx, self.lib, self._C = abi, ctx, ctx.lib, C
        self.rank, self.world, unique_id = _group_unique_id(ctx, rank, world, unique_id, dist_group)
        self.chain = engine.AoChain(ctx, ao_options)
        g = C.c_void_p()
        ctx._chk(self.lib.rfx_group_create(ctx.h, unique_id, self.rank, self.world, C.byref(g)))
        self.g = g
        ctx._chk(self.lib.rfx_group_attach_ao_chain(g, self.chain.h))
        ctx._chk(self.lib.rfx_group_set_rebalance(g, int(rebalance_every), int(rebalance_lag)))
        self.rebalance_every = rebalance_every
        self._host = None

    def render(self, cam_u, depth, velocity, normal=None, inp=None, out=None, stream=None):
        """Collective: one frame from full-frame device planes; this rank renders its band and joins the frame's collective."""
        f = self.chain._frame(cam_u, depth, velocity, normal, inp, out)
        self.ctx._chk(self.lib.rfx_ao_chain_render_sharded(self.chain.h, stream, self._C.byref(f)))

    def download_band(self, which: int = 1):
        """this rank's rows of AoChain output `which` of the last frame (numpy)"""
        b0, b1 = self.band_of_last_frame
        return self.chain.download(which)[b0:b1]

    def submit_host(self, *a, **k):
        raise self._abi.RfxError(f"rfx status {self._abi.ERR_UNSUPPORTED}: submit_host: the AO chain has no host-buffer path")


class InProcessAoGroup(InProcessGroup):
    """InProcessGroup for the AO chain (rfx_group_attach_ao_chains_inprocess): every member owns an AoChain with the same options."""

    def __init__(self, ctxs, ao_options, world: int):
        import ctypes as C

        from . import engine

        self._C, self.world = C, world
        self.ctxs = list(ctxs) if isinstance(ctxs, (list, tuple)) else [ctxs] * world
        assert len(self.ctxs) == world
        self.lib = self.ctxs[0].lib
        self.chains = [engine.AoChain(c, ao_options) for c in self.ctxs]
        self.groups = []
        for r, c in enumerate(self.ctxs):
            g = C.c_void_p()
            c._chk(self.lib.rfx_group_create_inprocess(c.h, r, world, C.byref(g)))
            self.groups.append(g)
        ga = (C.c_void_p * world)(*[g.value for g in self.groups])
        ca = (C.c_void_p * world)(*[ch.h.value for ch in self.chains])
        self.ctxs[0]._chk(self.lib.rfx_group_attach_ao_chains_inprocess(ga, ca, world))

    def render(self, cam_u, depth, velocity, normal=None, inp=None, out=None, wait: bool = True):
        """one frame: every member renders its band (its rows of `out` too); all of them finish before the next frame starts"""
        self._last_bounds = self.bounds
        for c, ch in zip(self.ctxs, self.chains):
            f = ch._frame(cam_u, depth, velocity, normal, inp, out)
            c._chk(self.lib.rfx_ao_chain_render_sharded(ch.h, None, self._C.byref(f)))
        if wait or len(set(self.ctxs)) > 1:
            for c in set(self.ctxs):
                c.sync()
