"""CPU tests of the multi-GPU host logic: the contiguous-band ShardPlan (halo recompute ranges) and the per-frame exchange of every
rank's band, exercised with world_size = 2 and 3 over gloo with the ORACLE standing in for the kernels (each "launch" commits only its row
range, like a row-sharded kernel).  The sharded result must equal the single-process chain bit for bit — if a halo were
one row short, a pass would read a stale row and the comparison would fail."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import chain_harness as ch
from realism_effects_b200 import abi
from realism_effects_b200.parallel import ShardPlan


def test_shard_plan_ranges():
    p = ShardPlan(2160, 8, 3, 4, 3.0)
    own = (810, 1080)
    k1, k2, p0, p1, p2, p3, k4 = p.ranges
    assert k4 == own and p3 == (809, 1081) and p2 == (805, 1085) and p1 == (801, 1089) and p0 == (797, 1093)
    assert k2 == (793, 1097) and k1 == (791, 1099)
    assert (p.r0, p.r1) == own
    overhead = sum(b - a for a, b in p.ranges) / (p.n_launches * (p.r1 - p.r0)) - 1.0  # extra rows launched / rows owned
    assert 0 < overhead < 0.15                                                    # the price of exchanging nothing per pass
    first, last = ShardPlan(2160, 8, 0, 4, 3.0), ShardPlan(2160, 8, 7, 4, 3.0)
    assert first.ranges[0][0] == 0 and last.ranges[0][1] == 2160                 # clipped at the frame border
    assert ShardPlan(2160, 1, 0, 4, 3.0).ranges == [(0, 2160)] * 7               # one GPU: whole planes
    assert ShardPlan(64, 2, 1, 0, 3.0).ranges == [(30, 64), (32, 64), (32, 64)]   # denoiseIterations = 0: K1, K2, K4 only
    assert len(ShardPlan(64, 2, 0, 2, 3.0, ssgi_mode=False).ranges) == 5          # SSR composes too (inputType specular)
    # the bands are a partition of the rows
    for world in (1, 2, 3, 4, 8):
        owned = [(p.r0, p.r1) for p in (ShardPlan(2160, world, r, 4, 3.0) for r in range(world))]
        assert owned[0][0] == 0 and owned[-1][1] == 2160 and all(a[1] == b[0] for a, b in zip(owned, owned[1:]))
    with pytest.raises(ValueError):
        ShardPlan(2161, 8, 0, 4, 3.0)
    assert ShardPlan(2160, 8, 0, 4, 11.0).poisson_halo == 12                      # demo radius 11 (SURVEY §8e)


def sharded_oracle_chain(inp, o, rank, world, all_gather_rows, bounds_per_frame=None, exchange_a=True):
    """The chain of chain_harness.run_oracle_chain, but every pass commits only its planned rows into this rank's planes, and
    all_gather_rows(plane, plan) completes a plane from the other ranks' bands after the frame.  bounds_per_frame: explicit band
    borders, one tuple per frame (the adaptive-band mode moves them between frames); None: equal bands.
    exchange_a: the A Poisson target's rows take part in the per-frame exchange like B's (what the native group does, by carrying a
    discarded texel from the rank that owns the row: DESIGN.md §5); False reproduces the pre-fix behaviour."""
    import orc

    H, W = inp.height, inp.width
    env = orc.Env(inp.env_map, inp.env_marginal, inp.env_conditional, inp.env_total)
    z32, z16 = (lambda: np.zeros((H, W, 4), np.float32)), (lambda: np.zeros((H, W, 4), np.float16))
    ssgi, tr, dnA, dnB, composed = z32(), [z32(), z32()], [z16(), z16()], [z16(), z16()], z32()
    keep_data, prev, bn_t, bn_p = 0.0, None, 0, 0

    def commit(dst, new, rng):
        dst[rng[0]:rng[1]] = new[rng[0]:rng[1]]

    for t, fr in enumerate(inp.frames):
        plan = ShardPlan(H, world, rank, 2 * o.denoise_iterations, o.radius, True, bounds=bounds_per_frame[t] if bounds_per_frame else None)
        rngs = iter(plan.ranges)
        cam = abi.make_camera(fr["cam"])
        bn_t = ch.next_blue(o.blue_noise_start, bn_t)
        sp = ch.ssgi_params(o, cam, bn_t, (inp.env_map.shape[1], inp.env_map.shape[0]))
        commit(ssgi, orc.ssgi_trace(sp, fr["depth"], fr["gbuffer"], None, fr["direct"], composed, env, inp.blue), next(rngs))
        prev = prev or fr["cam"]
        tp = ch.temporal_params(o, cam, fr["cam"]["position"], prev, keep_data, fr["moved"])
        t0, t1 = orc.temporal_reproject(tp, ssgi, fr["velocity"], dnB[0], dnB[1], tr[0], tr[1])
        r = next(rngs)
        commit(tr[0], t0, r)
        commit(tr[1], t1, r)
        keep_data, prev = 1.0, fr["cam"]
        for i in range(2 * o.denoise_iterations):
            horizontal = i % 2 == 0
            src = tr if i == 0 else (dnB if horizontal else dnA)
            dst = dnA if horizontal else dnB
            bn_p = ch.next_blue(o.blue_noise_start, bn_p)
            o0, o1 = orc.poisson_denoise(ch.poisson_params(o, bn_p, i == 0), fr["depth"], fr["gbuffer"], src[0], src[1], inp.blue, dst[0], dst[1])
            r = next(rngs)
            commit(dst[0], o0, r)
            commit(dst[1], o1, r)
        commit(composed, orc.gi_compose(ch.compose_params(cam), fr["depth"], fr["gbuffer"], dnB[0], dnB[1], composed), next(rngs))
        for plane in (composed, dnB[0], dnB[1]) + ((dnA[0], dnA[1]) if exchange_a else ()):
            all_gather_rows(plane, plan)
    return dict(composed=composed, dn0=dnB[0], dn1=dnB[1], tr0=tr[0], ssgi=ssgi, plan=plan)


def exchange_bands(plane, plan):
    """every rank's band of `plane` to every other rank (equal or unequal bands): what the native group's peer reads see after a frame"""
    mine = torch.from_numpy(np.ascontiguousarray(plane[plan.r0:plan.r1]).view(np.uint8).reshape(-1))
    reqs, theirs = [], {}
    for peer in range(plan.world):
        if peer != plan.rank:
            p0, p1 = plan.bounds[peer], plan.bounds[peer + 1]
            theirs[peer] = torch.empty((p1 - p0) * plane[0].nbytes, dtype=torch.uint8)
            reqs += [dist.isend(mine, peer), dist.irecv(theirs[peer], peer)]
    for r in reqs:
        r.wait()
    for peer, t in theirs.items():
        p0, p1 = plan.bounds[peer], plan.bounds[peer + 1]
        plane[p0:p1] = t.numpy().view(plane.dtype).reshape(p1 - p0, *plane.shape[1:])


def _worker(rank, world, port, q, bounds_per_frame):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OMP_NUM_THREADS="2")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        o = ch.Opts(steps=8, refine_steps=2, denoise_iterations=1)
        inp = ch.make_inputs(96, 64, 2)
        out = sharded_oracle_chain(inp, o, rank, world, exchange_bands, bounds_per_frame=bounds_per_frame)
        q.put((rank, {k: v.tobytes() for k, v in out.items() if k != "plan"}, (out["plan"].r0, out["plan"].r1)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("bounds_per_frame", [None, [(0, 16, 64)] * 2, [(0, 16, 64), (0, 48, 64)]],
                         ids=["equal-bands", "unequal-bands", "moving-bands"])  # moving: the adaptive mode moves the border between frames
def test_two_rank_sharded_bands_equal_single_process_bit_exact(bounds_per_frame):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, bounds_per_frame)) for r in range(2)]
    for p in procs:
        p.start()
    results = dict()
    for _ in procs:
        rank, planes, own = q.get(timeout=300)
        results[rank] = (planes, own)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    o = ch.Opts(steps=8, refine_steps=2, denoise_iterations=1)
    inp = ch.make_inputs(96, 64, 2)
    ref = ch.run_oracle_chain(inp, o)[-1]
    for rank, (planes, (r0, r1)) in results.items():
        for k in ("composed", "dn0", "dn1"):                       # exchanged planes: the whole frame must match on every rank
            assert planes[k] == ref[k].tobytes(), (rank, k)
        for k in ("tr0", "ssgi"):                                  # not exchanged: this rank's own rows must match
            got = np.frombuffer(planes[k], ref[k].dtype).reshape(ref[k].shape)
            assert got[r0:r1].tobytes() == ref[k][r0:r1].tobytes(), (rank, k)


def _worker3(rank, world, port, q, exchange_a):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OMP_NUM_THREADS="2")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        o = ch.Opts(steps=6, refine_steps=1, denoise_iterations=2)
        inp = ch.make_inputs(*WIDE_CASE, fov=75.0)
        out = sharded_oracle_chain(inp, o, rank, world, exchange_bands, exchange_a=exchange_a)
        q.put((rank, {k: v.tobytes() for k, v in out.items() if k != "plan"}))
    finally:
        dist.destroy_process_group()


WIDE_CASE = (112, 144, 4)  # width, height, frames (fov 75 below: the sky's silhouette runs through the upper band border)


def _run3(exchange_a):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker3, args=(r, 3, port, q, exchange_a)) for r in range(3)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return res


def test_three_ranks_two_denoise_iterations_with_the_a_target_taken_from_its_owner():
    """world_size 3, denoiseIterations 2 (four Poisson passes: the A target is written twice per frame on shrinking row ranges).  A pixel the
    shader discards keeps its A texel, and the LINEAR taps of the next pass read it at silhouettes; on rows outside a rank's last A range the
    local texel is the wrong pass's.  With the A rows coming from their owner every frame (the rule the native group implements by carrying the
    texel from the owning rank) every rank's frame equals the single-process chain bit for bit.  The failure without the rule needs a pixel
    that turns from shaded to discarded between two frames right at a band border; this small scene does not have one — the bench frame does:
    tools/emulate_group_cpu.py reproduces there, pixel for pixel, what the N = 4 GPU run showed (profiles/r02_group_a_target_cpu_emulation.txt)."""
    o = ch.Opts(steps=6, refine_steps=1, denoise_iterations=2)
    inp = ch.make_inputs(*WIDE_CASE, fov=75.0)
    ref = ch.run_oracle_chain(inp, o)[-1]
    good = _run3(True)
    for rank, planes in good.items():
        for k in ("composed", "dn0", "dn1"):
            assert planes[k] == ref[k].tobytes(), (rank, k)


def test_host_path_row_sets_cover_what_each_launch_reads():
    """ShardPlan.local_input_rows (G-buffer / direct-light rows a rank uploads) contains every launch's output rows plus the
    rows its Poisson taps and quad helpers reach; the ranks' own bands (uploaded + all-gathered depth / velocity) tile the frame.
    Equal bands, and the bands one rebalancing step makes of them when the cost grows down the frame."""
    from realism_effects_b200.parallel import ShardPlan, rebalance

    for world, H, radius, iters in ((2, 128, 3.0, 1), (2, 4320, 8.0, 2), (8, 17280, 8.0, 2), (4, 960, 12.5, 3)):
        equal = ShardPlan(H, world, 0, 2 * iters, radius).bounds
        for bounds in (equal, rebalance(equal, [1.0 + 2.0 * r for r in range(world)])):
            covered = np.zeros(H, np.int32)
            for rank in range(world):
                p = ShardPlan(H, world, rank, 2 * iters, radius, True, bounds=bounds)
                a, b = p.r0, p.r1
                la, lb = p.local_input_rows
                covered[a:b] += 1
                assert la <= a and lb >= b
                for k, (r0, r1) in enumerate(p.ranges):
                    reach = p.poisson_halo if 2 <= k < 2 + p.n_poisson_passes else 0   # K3 passes read G-buffer rows around their output
                    assert la <= max(0, r0 - reach) and lb >= min(H, r1 + reach), (world, bounds, rank, k)
            assert (covered == 1).all()


def test_rebalance_moves_borders_towards_equal_cost():
    from realism_effects_b200.parallel import ShardPlan, rebalance

    H, n = 17280, 8
    density = lambda r: 0.2 + 2.0 * np.exp(-((r / H - 0.55) ** 2) / 0.02) + 0.8 * (r > 0.7 * H)  # noqa: E731  cheap sky, expensive horizon, floor
    rows = density(np.arange(H))
    cost = lambda b: [float(rows[b[i]:b[i + 1]].sum()) for i in range(n)]  # noqa: E731
    b = tuple(H * i // n for i in range(n + 1))
    spread0 = max(cost(b)) / (sum(cost(b)) / n)
    for _ in range(12):
        nb = rebalance(b, cost(b))
        assert nb[0] == 0 and nb[-1] == H and all(x % 16 == 0 for x in nb) and all(nb[i + 1] - nb[i] >= 64 for i in range(n))
        assert nb == rebalance(b, cost(b))                                   # deterministic
        ShardPlan(H, n, 3, 4, 8.0, True, bounds=nb)                           # always a valid plan
        b = nb
    spread = max(cost(b)) / (sum(cost(b)) / n)
    assert spread0 > 1.5 and spread < 1.06, (spread0, spread)                  # max-over-ranks within 6 % of the mean
    # measurements taken with older borders are interpreted on those borders
    assert rebalance((0, 1000, 2000), [3.0, 1.0], measured_bounds=(0, 1200, 2000), align=8, damping=1.0) == (0, 800, 2000)
    # a rank that reports (almost) nothing cannot collapse to less than min_rows, nor can a band exceed max_share x the mean
    assert rebalance((0, 1024, 2048), [1e-12, 5.0], min_rows=64, damping=1.0)[1] <= 2048 - 64
    with pytest.raises(ValueError):
        ShardPlan(128, 2, 0, 2, 3.0, True, bounds=(0, 64, 100))


def test_rebalance_caps_every_band_including_the_last():
    """Cost concentrated in the lower rows (cheap sky on top = the LAST band): no band, the last one included, may exceed
    max_share x the mean height — the host path sizes its read-back staging by that bound."""
    from realism_effects_b200.parallel import rebalance

    H, n = 2160, 8
    rows = np.where(np.arange(H) < 0.35 * H, 10.0, 0.01)
    cost = lambda b: [float(rows[b[i]:b[i + 1]].sum()) for i in range(n)]  # noqa: E731
    b = tuple(H * i // n // 16 * 16 for i in range(n)) + (H,)
    cap = int(4.0 * H / n)
    for share in (4.0, 1.5):
        bb = b
        for _ in range(40):
            bb = rebalance(bb, cost(bb), max_share=share)
            assert all(bb[i + 1] - bb[i] <= max(64, int(share * H / n)) for i in range(n)), (share, bb)
            assert bb[0] == 0 and bb[-1] == H and all(bb[i + 1] - bb[i] >= 64 for i in range(n))
    assert cap == 1080


def test_portrait_frames_reach_further_in_rows():
    """The Poisson offset is rotated after the division by the resolution, so for H > W a tap reaches radius * H / W rows."""
    assert ShardPlan(960, 2, 0, 2, 3.0, True, bounds=(0, 480, 960), width=540).poisson_halo == 7   # ceil(3 * 960 / 540) + 1
    assert ShardPlan(540, 2, 0, 2, 3.0, True, bounds=(0, 272, 540), width=960).poisson_halo == 4   # landscape: unchanged
    # brute force over the tap geometry of poisson_denoise.frag:177-189 (flatness = 1, any rotation)
    W, H, radius = 540, 960, 3.0
    SQ = 2 ** 0.5
    taps = [(-1, 0), (0, -1), (1, 0), (0, 1), (-.25 * SQ, -.25 * SQ), (.25 * SQ, -.25 * SQ), (.25 * SQ, .25 * SQ), (-.25 * SQ, .25 * SQ)]
    reach = 0.0
    for ang in np.linspace(0, 2 * np.pi, 721):
        s_, c_ = np.sin(ang), np.cos(ang)
        for px, py in taps:
            ox, oy = radius * px / W, radius * py / H
            reach = max(reach, abs((-s_ * ox + c_ * oy) * H))
    assert 5.0 < reach <= ShardPlan(H, 2, 0, 2, radius, True, bounds=(0, 480, 960), width=W).poisson_halo - 1


def test_native_shard_arithmetic_matches_the_python_mirror(built):
    """rfx_shard_ranges / rfx_shard_rebalance (csrc/rfx_group.inl, what the product path uses) == ShardPlan / rebalance."""
    import ctypes as C

    from realism_effects_b200.parallel import rebalance

    lib = abi.lib()
    rng = np.random.default_rng(7)
    for W, H, world, passes, radius, ssgi in ((3840, 2160, 8, 4, 3.0, True), (540, 960, 2, 2, 3.0, True), (7680, 4320, 8, 4, 11.0, True),
                                              (256, 128, 2, 0, 3.0, True), (640, 360, 4, 2, 2.5, False)):
        bounds = tuple(int(round(H * i / world / 16.0)) * 16 for i in range(world)) + (H,)
        for rank in range(world):
            p = ShardPlan(H, world, rank, passes, radius, ssgi, bounds=bounds, width=W)
            n = p.n_launches
            out = (C.c_uint32 * (2 * n))()
            assert lib.rfx_shard_ranges(W, H, p.r0, p.r1, passes, radius, int(ssgi), out, n) == 0
            assert [(out[2 * k], out[2 * k + 1]) for k in range(n)] == p.ranges, (W, H, rank)
        b = bounds
        for _ in range(6):
            costs = [float(x) for x in rng.uniform(0.2, 3.0, world)]
            cb = (C.c_uint32 * (world + 1))(*b)
            cc = (C.c_float * world)(*costs)
            co = (C.c_uint32 * (world + 1))()
            assert lib.rfx_shard_rebalance(cb, None, cc, world, co) == 0
            costs32 = [float(np.float32(c)) for c in costs]
            want = rebalance(b, costs32) if H >= world * 64 else None
            if want is not None:
                assert tuple(co) == want, (b, costs, tuple(co), want)
                b = want
    assert lib.rfx_shard_ranges(64, 64, 10, 10, 2, 3.0, 1, (C.c_uint32 * 10)(), 5) != 0     # empty band
    assert lib.rfx_shard_ranges(64, 64, 0, 32, 2, 3.0, 1, (C.c_uint32 * 10)(), 4) != 0      # wrong launch count
