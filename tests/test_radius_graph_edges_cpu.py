"""Hand-placed event streams at the radius graph's decision edges, and the build kernel's per-voxel regimes they reach.

tests/test_radius_graph_edges_gpu.py runs every case of CASES through dagr_graph_sort, dagr_l1_build and dagr_graph_export and
compares the edge_index with the graph oracle bit for bit.  The cases are built here, in numpy, and checked without a GPU:
  * each case's intended pairs are edges, or not, in oracle.ref_ops.RefGraph (graph_oracle.c): the time rule dt <= delta_t,
    the Chebyshev radius r, the K cap (spiral order, then the newest FIFO entry), the FIFO depth Q and the sensor border;
  * each case reaches the kernel regimes it names, restated from csrc/build_l1.cu by regimes(): time-bucket pruning or not
    (staged, the voxel's new events span fewer than 8 slices, the sort's flag clear), the ring walk or the cell walk
    (TW <= 32 && TH <= 32 && r <= 8), the cooperative continuation (cell walk with ncell > BL_R1 = 96) and the staging class
    of the 3x3 neighbourhood (lean / regular / dense / global, from the DAGR_L1_* capacities).  Every claimed regime must
    hold at least one voxel with new events, so the coverage cannot move silently;
  * the sort's time-order flag model (tests/test_graph_sort_cpu.py: ref_sort) on hand cases: it is clear only where the
    clamped samples come as ascending contiguous runs in arrival order, each time-sorted.

Times are the kernels' int32 microseconds; slices are C quotients t / max(delta_t, 1) (truncated toward zero).
"""
import numpy as np
import pytest
import torch

from tests.test_graph_sort_cpu import clamp_xyb, ref_sort
from tests.test_l1_kernels_cpu import l1_caps, oracle_edges, voxel_stats

BL_NB, BL_R1 = 8, 96
T24 = 1 << 24


class Case:
    """one hand-placed stream: geometry arguments, events in arrival order, intended (src, dst, is_edge) pairs, claims"""

    def __init__(self, W, H, B=1, radius=0.01, T=1_000_000, K=16, Q=128, claims=(), min_idx=0, time_sorted=True):
        self.geo = dict(W=W, H=H, B=B, radius=radius, T=T, K=K, Q=Q)
        self.claims, self.min_idx, self.time_sorted = set(claims), min_idx, time_sorted
        self.ev = []                                        # (t, x, y, b) in creation order
        self.pairs = []

    def add(self, x, y, t, b=0):
        self.ev.append((int(t), int(x), int(y), int(b)))
        return len(self.ev) - 1

    def pair(self, src, dst, edge):
        self.pairs.append((src, dst, bool(edge)))

    def geometry(self, device="cpu"):
        from dagr_b200.geometry import Geometry
        g = self.geo
        return Geometry(g["W"], g["H"], g["B"], radius=g["radius"], time_window=g["T"], max_neighbors=g["K"],
                        max_queue_size=g["Q"], device=device)

    def arrays(self):
        """(batch int32[N], pos int32[N, 3]) in arrival order: a stable sort by t (time_sorted), else the creation order"""
        ev = np.array(self.ev, np.int64).reshape(-1, 4)
        order = np.argsort(ev[:, 0], kind="stable") if self.time_sorted else np.arange(len(ev))
        self.order = np.asarray(order)
        arr = np.empty(len(ev), np.int64)
        arr[self.order] = np.arange(len(ev))
        self.arrival = arr
        ev = ev[self.order]
        # contiguous: the kernels read the arrays through their data pointers
        return (torch.from_numpy(np.ascontiguousarray(ev[:, 3], np.int32)), torch.from_numpy(np.ascontiguousarray(ev[:, [1, 2, 0]], np.int32)))

    def arrival_pairs(self):
        return [(int(self.arrival[s]), int(self.arrival[d]), e) for s, d, e in self.pairs]


def slices(t, d):
    """C quotient t / d (truncation toward zero), as bl_div"""
    t = np.asarray(t, np.int64)
    return np.sign(t) * (np.abs(t) // d)


def regimes(geom, batch, pos, min_idx=0):
    """boolean masks over the pool1 voxels (with new events) of the regimes dagr_l1_build runs on them, flags from the sort"""
    batch, pos = np.asarray(batch, np.int64), np.asarray(pos, np.int64).reshape(-1, 3)
    r = ref_sort(geom, batch, pos, np.zeros(len(batch), np.float32))
    caps = l1_caps()
    nown, total = voxel_stats(geom, r["start"])
    x, y, b = clamp_xyb(geom, batch, pos)
    lv = geom.levels[0]
    cx, cy = lv.cellx.numpy()[x].astype(np.int64), lv.celly.numpy()[y].astype(np.int64)
    cell = (b * geom.ny1 + cy) * geom.nx1 + cx
    cells = geom.B * geom.ny1 * geom.nx1
    new = np.arange(len(batch)) >= min_idx
    sl = slices(pos[:, 2], max(geom.dt_us, 1))
    smin = np.full(cells, np.iinfo(np.int64).max)
    smax = np.full(cells, np.iinfo(np.int64).min)
    np.minimum.at(smin, cell[new], sl[new])
    np.maximum.at(smax, cell[new], sl[new])
    has = np.zeros(cells, bool)
    has[cell[new]] = True
    short = has & (smax - (smin - 1) < BL_NB)
    vx0, vy0 = geom.vx0.numpy().astype(np.int64), geom.vy0.numpy().astype(np.int64)
    tw = np.tile(np.diff(vx0)[None, :], (geom.ny1, 1)).ravel() + 2 * geom.r
    th = np.tile(np.diff(vy0)[:, None], (1, geom.nx1)).ravel() + 2 * geom.r
    rings = np.tile((tw <= 32) & (th <= 32), geom.B) & (geom.r <= 8)
    L, R, D = caps["BUILD_LEAN"], caps["BUILD"], caps["BUILD_DENSE"]
    pr = short & (total <= D) & (not r["flag"])             # pruned in the defer = 1 launch (staged up to the dense capacity)
    return dict(flag=r["flag"], pruned=pr, unpruned=has & ~pr, rings=has & rings, cells=has & ~rings,
                coop=has & ~rings & (geom.ncell > BL_R1), lean=has & (total <= L), regular=has & (total > L) & (total <= R),
                dense=has & (total > R) & (total <= D), **{"global": has & (total > D)})


# ------------------------------------------------------------------------------------------------------------------------
# case builders
# ------------------------------------------------------------------------------------------------------------------------
def _slots(geom, every=3, margin=1):
    """top-left pixels of pool1 voxels (every `every`-th column and row, away from the grid edge): disjoint 3x3 neighbourhoods"""
    vx0, vy0 = geom.vx0.tolist(), geom.vy0.tolist()
    return [(cx, cy, vx0[cx], vy0[cy]) for cy in range(margin, geom.ny1 - margin, every) for cx in range(margin, geom.nx1 - margin, every)]


def _filler(c, geom, cx, cy, n, t_lo, t_hi, rng):
    """n events in each of the 8 voxels around (cx, cy), times in [t_lo, t_hi): older than everything probed there"""
    vx0, vy0 = geom.vx0.tolist(), geom.vy0.tolist()
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx or dy:
                X, Y = cx + dx, cy + dy
                xs = rng.integers(vx0[X], vx0[X + 1], n)
                ys = rng.integers(vy0[Y], vy0[Y + 1], n)
                for x, y, t in zip(xs, ys, np.sort(rng.integers(t_lo, t_hi, n))):
                    c.add(x, y, t)


def time_case(radius=0.01, T=1_000_000, W=240, H=180, fill=0, anchors=None, dts=None, claims=("pruned",), time_sorted=True):
    """pairs (src, dst) at dt = t_dst - t_src in dts around each anchor A: t_src in {A - 1, A, A + 1}; the four pairs of one
    (anchor, offset) share one voxel (src at (X0 + k, Y0), dst at (X0 + k, Y0 + 1)); fill: events in each of the 8 voxels around
    it, older than every pair by more than delta_t (their records clamp into bucket 0)"""
    c = Case(W, H, radius=radius, T=T, claims=claims, time_sorted=time_sorted)
    geom = c.geometry()
    D, d = geom.dt_us, max(geom.dt_us, 1)
    if anchors is None:
        anchors = [50 * d, (T24 // d) * d, T24, -5 * d, 0]
    if dts is None:
        dts = sorted({0, max(D - 1, 0), D, D + 1})
    rng = np.random.default_rng(D + fill)
    slots = iter(_slots(geom))
    t_first = min(anchors) - 1
    for A in anchors:
        for a in (-1, 0, 1):
            cx, cy, X0, Y0 = next(slots)
            if fill:
                _filler(c, geom, cx, cy, fill, t_first - 60 * d, t_first - 3 * d, rng)
            for k, dt in enumerate(dts):
                s = c.add(X0 + k, Y0, A + a)
                e = c.add(X0 + k, Y0 + 1, A + a + dt)
                c.pair(s, e, dt <= D)
    return c


def span_case():
    """a voxel whose new events span exactly 7 slices (pruned) and one spanning 8 (not pruned): one event per slice, alternating
    between two neighbouring pixels; consecutive events are delta_t apart (edges), the next but one 2 delta_t (none).  A
    neighbouring voxel holds records older than sbase (bucket 0 after clamping), one exactly delta_t before the first event,
    and records newer than every event of the voxel (bucket 7 after clamping, arriving later)"""
    c = Case(240, 180, claims=("pruned", "unpruned"))
    geom = c.geometry()
    d = geom.dt_us
    (_, _, X0, Y0), (_, _, X1, Y1) = _slots(geom)[5], _slots(geom)[40]
    for (X, Y), n in (((X0, Y0), 7), ((X1, Y1), 8)):
        t0 = 40 * d + 3
        ids = [c.add(X + 1 + (j & 1), Y + 1, t0 + j * d) for j in range(n)]
        for j in range(n - 1):
            c.pair(ids[j], ids[j + 1], True)
            if j + 2 < n:
                c.pair(ids[j], ids[j + 2], False)
        old = [c.add(X - 1, Y + 1, t0 - k * d - o) for k, o in ((30, 0), (2, 1), (2, 0), (1, 1), (1, 0))]
        for o, e in zip(old, (False, False, False, False, True)):
            c.pair(o, ids[0], e)
        c.add(X - 1, Y + 2, t0 + 20 * d)
        c.add(X - 1, Y + 3, t0 + 9 * d)
    return c


def incremental_case():
    """min_idx > 0: old events (arrival < min_idx) in the same voxel as the new ones, far in the past and exactly delta_t before
    the oldest new event; smin comes from the new events only, so the voxel is pruned"""
    c = Case(240, 180, claims=("pruned",))
    geom = c.geometry()
    d = geom.dt_us
    pairs = []
    for i, (_, _, X, Y) in enumerate(_slots(geom)[:6]):
        t0 = 70 * d + (i - 1)                                       # the oldest new event at kd - 1, kd, kd + 1, ...
        far = c.add(X, Y, t0 - 40 * d)
        at = c.add(X + 1, Y, t0 - d)
        just = c.add(X + 2, Y, t0 - d - 1)
        pairs.append((far, at, just, X, Y, t0))
    m = len(c.ev)
    for far, at, just, X, Y, t0 in pairs:
        n0 = c.add(X + 1, Y + 1, t0)
        n1 = c.add(X, Y + 1, t0 + 3 * d)
        c.pair(far, n0, False); c.pair(at, n0, True); c.pair(just, n0, False); c.pair(at, n1, False)
    c.min_idx = m
    return c


def _inversion(B, batch_ids, between=False):
    """the dropped-edge example: (100, 100) at t = 990000, then (101, 100) at t = 960000 (dt = -30000 <= delta_t: an edge)"""
    c = Case(240, 180, B=B, claims=("unpruned",), time_sorted=False)
    a = c.add(100, 100, 990000, batch_ids[0])
    if between:
        c.add(50, 50, 970000, 1)
    e = c.add(101, 100, 960000, batch_ids[1])
    c.pair(a, e, True)
    return c


def order_cases():
    out = {}
    out["order-inversion-across-pixels-B1"] = _inversion(1, (0, 0))
    out["order-interleaved-samples-B2"] = _inversion(2, (0, 0), between=True)
    out["order-batch-ids-clamped-into-one-sample-B2"] = _inversion(2, (1, 7))
    c = Case(240, 180, claims=("unpruned",), time_sorted=False)
    a = c.add(100, 100, 990000)
    e = c.add(100, 100, 960000)
    c.pair(a, e, True)
    out["order-inversion-inside-a-pixel"] = c
    c = Case(240, 180, claims=("pruned",))
    rng = np.random.default_rng(5)
    ids = [c.add(x, y, 500000) for x, y in zip(rng.integers(60, 75, 300), rng.integers(60, 75, 300))]
    c.pair(ids[0], ids[1], max(abs(c.ev[0][1] - c.ev[1][1]), abs(c.ev[0][2] - c.ev[1][2])) <= 3)
    out["order-all-times-equal"] = c
    # the same inversion hidden by an id below 0 (-3 is sample 0)
    c = Case(240, 180, B=2, claims=("unpruned",), time_sorted=False)
    a = c.add(30, 30, 990000, -3)
    e = c.add(31, 30, 960000, 0)
    c.pair(a, e, True)
    out["order-negative-id-clamped-to-0-B2"] = c
    return out


DIRS = [(1, 0), (1, 1), (0, 1), (-1, 1), (-1, 0), (-1, -1), (0, -1), (1, -1)]


def chebyshev_case(radius=0.01, W=240, H=180):
    """centres with neighbours at Chebyshev distance r (edges) and r + 1 (none) in all eight directions; the centre is newest"""
    c = Case(W, H, radius=radius, claims=("pruned",))
    geom = c.geometry()
    r = geom.r
    step = 4 * r + 6
    for i, (x0, y0) in enumerate([(step, step), (2 * step + 1, step + 2), (step + 3, 2 * step + 1)]):
        t = 300000 + 100 * i
        nb = [(c.add(x0 + dx * dd, y0 + dy * dd, t + k), dd == r) for k, (dd, (dx, dy)) in enumerate((dd, v) for dd in (r, r + 1) for v in DIRS)]
        ctr = c.add(x0, y0, t + 50)
        for n, e in nb:
            c.pair(n, ctr, e)
    return c


def border_case():
    """sensor corners and edges: the probe's window leaves the sensor (the reference's break at a pixel outside it)"""
    c = Case(240, 180, claims=("pruned",))
    W, H = 240, 180
    t = 200000
    for (x, y) in [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (120, 0), (120, H - 1), (0, 90), (W - 1, 90)]:
        sx, sy = (1 if x == 0 else -1 if x == W - 1 else 0), (1 if y == 0 else -1 if y == H - 1 else 0)
        inner = [c.add(x + sx * k, y + sy * k, t + k) for k in (1, 2, 3)] + [c.add(x + (sx or 1) * 2, y + (sy or 1), t + 4)]
        edge = c.add(x, y, t + 9)
        for n in inner:
            c.pair(n, edge, True)
        c.pair(edge, inner[0], False)                               # the older arrival never reads a newer one
        t += 20
    return c


def voxel_border_case():
    """a centre in the middle of a voxel and one neighbour in each of the 8 voxels around it (every cellmask bit), in an
    interior voxel and in the four corner voxels of the grid"""
    c = Case(240, 180, claims=("pruned",))
    geom = c.geometry()
    vx0, vy0 = geom.vx0.tolist(), geom.vy0.tolist()
    t = 100000
    for cx, cy in [(10, 10), (0, 0), (geom.nx1 - 1, 0), (0, geom.ny1 - 1), (geom.nx1 - 1, geom.ny1 - 1), (20, 13)]:
        X0, X1, Y0, Y1 = vx0[cx], vx0[cx + 1], vy0[cy], vy0[cy + 1]
        mx, my = X0 + 2, Y0 + 2
        nb = []
        for y in (Y0 - 1, my, Y1):
            for x in (X0 - 1, mx, X1):
                if (x, y) != (mx, my) and 0 <= x < geom.W and 0 <= y < geom.H:
                    nb.append(c.add(x, y, t + len(nb)))
        ctr = c.add(mx, my, t + 20)
        for n in nb:
            c.pair(n, ctr, True)
        t += 50
    return c


WALKS = {   # name: (W, H, radius, claims)
    "r8-rings": (640, 480, 7.5 / 640, {"rings"}),
    "r9-cells": (640, 480, 8.5 / 640, {"cells", "coop"}),
    "tw32-33-both-walks": (1280, 720, 4.5 / 1280, {"rings", "cells", "coop"}),
    "ncell81-rings": (640, 480, 3.5 / 640, {"rings"}),
    "ncell121-rings": (640, 480, 4.5 / 640, {"rings"}),
    "ncell81-cells": (1600, 480, 3.5 / 1600, {"cells"}),
    "ncell121-cells-coop": (1600, 480, 4.5 / 1600, {"cells", "coop"}),
}


def walk_case(name, long_span):
    """a sparse background (unsaturated events: the walks run to the end, the continuation runs) and a dense cluster (K cap)
    in a region of the sensor; times over 1 s (not pruned) or over min(50 ms, 6 delta_t) (pruned)"""
    W, H, radius, claims = WALKS[name]
    c = Case(W, H, radius=radius, claims=claims | {"unpruned" if long_span else "pruned"})
    geom = c.geometry()
    span = 1_000_000 if long_span else min(50_000, 6 * geom.dt_us)
    rng = np.random.default_rng(len(name) + long_span)
    n_bg, n_cl = 2500, 1500
    x = np.concatenate([rng.integers(0, W // 2, n_bg), rng.integers(W // 4, W // 4 + 3 * geom.r, n_cl)])
    y = np.concatenate([rng.integers(0, H // 2, n_bg), rng.integers(H // 4, H // 4 + 3 * geom.r, n_cl)])
    for xx, yy, tt in zip(x, y, rng.integers(0, span, n_bg + n_cl)):
        c.add(xx, yy, 1_000_000 - span + tt)
    return c


def k_case(K):
    """K - 1, K and K + 1 candidates around three centres: two records per spiral cell (cell 0 = the centre's own pixel); the
    centre keeps the first K - 1 in spiral order, the newer record of a cell first"""
    c = Case(240, 180, K=K, claims=("pruned",))
    geom = c.geometry()
    sp = geom.spiral.tolist()
    t = 400000
    for i, n in enumerate((K - 1, K, K + 1)):
        x0, y0 = 40 + 40 * i, 60
        recs = []
        for j in range(n):
            dx, dy = sp[j // 2]
            recs.append((j // 2, j % 2, c.add(x0 + dx, y0 + dy, t + j)))
        ctr = c.add(x0, y0, t + 40)
        order = sorted(recs, key=lambda v: (v[0], -v[1]))            # spiral cell, then the newer record
        for k, (_, _, rid) in enumerate(order):
            c.pair(rid, ctr, k < K - 1)
        t += 100
    return c


def q_case(Q):
    """Q - 1, Q and Q + 1 events on a pixel (the FIFO keeps the newest Q): with Q + 1 the oldest is invisible to every probe"""
    c = Case(240, 180, Q=Q, claims=("pruned",))
    t = 600000
    for i, n in enumerate((Q - 1, Q, Q + 1)):
        x0, y0 = 40 + 40 * i, 100
        ids = [c.add(x0, y0, t + j) for j in range(n)]
        probe = c.add(x0 + 1, y0, t + n + 5)
        if n >= 2:
            c.pair(ids[0], ids[1], n <= Q)
        if n >= 1:
            c.pair(ids[-1], probe, True)
            if n >= 16:
                c.pair(ids[-16], probe, False)                     # K = 16: the 15 newest only
        t += 1000
    return c


def hot_pixel_case():
    """200 events on one pixel (Q = 128) whose times straddle a slice boundary, probed from the next pixel"""
    c = Case(240, 180, claims=("pruned",))
    d = c.geometry().dt_us
    t0 = 60 * d - 100
    ids = [c.add(77, 77, t0 + j) for j in range(200)]
    probe = c.add(78, 77, t0 + 250)
    c.pair(ids[0], ids[1], False)                                  # ids[0..71] left the FIFO
    c.pair(ids[71], ids[72], False)
    c.pair(ids[72], ids[73], True)
    c.pair(ids[-1], probe, True)
    return c


def _cases():
    out = {}
    for name, kw in [("time-d10000", {}), ("time-d13281-r9", dict(radius=8.5 / 640, W=640, H=480, claims=("pruned", "cells", "coop"))),
                     ("time-d1", dict(T=100)), ("time-d0", dict(T=50))]:
        out[name] = lambda kw=kw: time_case(**kw)
    out["time-d10000-dt-minus-1"] = lambda: time_case(dts=[-1], claims=("unpruned",), time_sorted=False)
    # one time case in each staging class: 150 / 220 / 600 / 1600 records in each of the 8 voxels around a pair voxel put its
    # 3x3 neighbourhood at ~1200 (lean), ~1770 (regular), ~4800 (dense) and ~12800 records (global, never pruned)
    for cls, fill in (("lean", 150), ("regular", 220), ("dense", 600), ("global", 1600)):
        out[f"time-d10000-staging-{cls}"] = lambda cls=cls, fill=fill: time_case(
            fill=fill, anchors=[50 * 10000, T24], claims=(cls, "unpruned" if cls == "global" else "pruned"))
    out["buckets-span-7-and-8"] = span_case
    out["buckets-incremental-min-idx"] = incremental_case
    for name, c in order_cases().items():
        out[name] = lambda c=c: c
    out["space-chebyshev-r-and-r+1"] = chebyshev_case
    out["space-chebyshev-r8"] = lambda: chebyshev_case(7.5 / 640, 640, 480)
    out["space-sensor-border"] = border_case
    out["space-voxel-borders"] = voxel_border_case
    for name in WALKS:
        for long_span in (False, True):
            out[f"walk-{name}-{'1s' if long_span else '50ms'}"] = lambda name=name, ls=long_span: walk_case(name, ls)
    for K in (1, 8, 16):
        out[f"k-cap-K{K}"] = lambda K=K: k_case(K)
    for Q in (1, 128, 255):
        out[f"fifo-Q{Q}"] = lambda Q=Q: q_case(Q)
    out["fifo-hot-pixel-over-Q-straddling-a-bucket"] = hot_pixel_case
    return out


CASES = _cases()
CLAIMS = {"pruned", "unpruned", "rings", "cells", "coop", "lean", "regular", "dense", "global"}


def build_case(name):
    c = CASES[name]()
    c.batch, c.pos = c.arrays()
    return c


def oracle_batch(geom, batch):
    """the oracle has no semantics for out-of-range sample ids: it runs on the ids the kernels clamp to"""
    return batch.clamp(0, geom.B - 1)


# ------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_case_pairs_and_regimes(name):
    c = build_case(name)
    geom = c.geometry()
    assert c.claims <= CLAIMS and (c.pairs or name.startswith("walk-")), name      # the walks' streams are random
    edges = oracle_edges(geom, oracle_batch(geom, c.batch), c.pos)
    have = set(zip(edges[0].tolist(), edges[1].tolist()))
    for s, d, e in c.arrival_pairs():
        assert ((s, d) in have) == e, (name, s, d, e)
    reg = regimes(geom, c.batch.numpy(), c.pos.numpy(), c.min_idx)
    for k in c.claims:
        assert reg[k].any(), (name, k)
    if not c.time_sorted:
        assert reg["flag"] and not reg["pruned"].any(), name


def test_time_cases_reach_the_bucket_edges():
    """slice boundaries kD - 1, kD, kD + 1 on both sides of 2^24 (bl_div's two arms), negative times and times across 0"""
    for name in ("time-d10000", "time-d13281-r9", "time-d1"):
        c = build_case(name)
        geom = c.geometry()
        d = geom.dt_us
        t = c.pos[:, 2].numpy().astype(np.int64)
        assert d < 3 or {0, 1, d - 1} <= set((t % d).tolist()), name
        assert (t < T24).any() and (t >= T24).any() and (t == T24 - 1).any() and (t == T24).any(), name
        assert (t < 0).any() and (t == 0).any() and (t == 1).any() and (t == -1).any(), name
    assert build_case("time-d13281-r9").geometry().dt_us == 13281
    assert build_case("time-d1").geometry().dt_us == 1 and build_case("time-d0").geometry().dt_us == 0


def test_slices_truncate_toward_zero():
    assert slices([-10001, -10000, -9999, -1, 0, 1, 9999, 10000, T24 + 5], 10000).tolist() == [-1, -1, 0, 0, 0, 0, 0, 1, 1677]


def test_span_case_prunes_7_slices_and_not_8():
    c = build_case("buckets-span-7-and-8")
    geom = c.geometry()
    reg = regimes(geom, c.batch.numpy(), c.pos.numpy())
    lv = geom.levels[0]
    vox = [int(lv.celly[c.pos[i, 1]]) * geom.nx1 + int(lv.cellx[c.pos[i, 0]]) for i in (c.arrival[0], c.arrival[14])]
    assert reg["pruned"][vox[0]] and reg["unpruned"][vox[1]]


def test_flag_model_on_hand_cases():
    """ref_sort's flag: clamped samples as ascending contiguous runs, each time-sorted"""
    from dagr_b200.geometry import Geometry
    geom = Geometry(240, 180, 3, device="cpu")

    def flag(batch, t):
        pos = np.stack([np.full(len(t), 5), np.full(len(t), 5), t], 1)
        return ref_sort(geom, np.asarray(batch), pos, np.zeros(len(t), np.float32))["flag"]
    assert not flag([0, 0, 1, 1, 2], [5, 6, 1, 1, 0])              # drops between contiguous ascending samples
    assert flag([0, 0, 1, 1, 2], [5, 6, 2, 1, 0])                  # an inversion inside sample 1
    assert flag([0, 1, 0], [1, 2, 3])                              # interleaved: time order not proven
    assert flag([1, 0], [1, 2])                                    # descending samples
    assert not flag([2, 9, 2], [5, 6, 7]) and flag([2, 9, 2], [5, 7, 6])   # 9 clamps to 2: one sample, whose times must ascend
    assert flag([2, 7], [990000, 960000])                          # raw ids differ, clamped ids do not
    assert not flag([-1, 0, 1], [3, 4, 0]) and flag([-1, 0, 1], [4, 3, 0])
    assert not flag([0], [7]) and not flag([0, 0, 0], [7, 7, 7])
