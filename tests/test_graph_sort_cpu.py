"""The graph sort's, the streaming rings' and the edge exporter's numpy models, checked without a GPU.

tests/test_graph_sort_gpu.py runs every entry point of csrc/graph.cu through the C-ABI and compares its outputs bit for bit with
the models below:
  * ref_sort: the counting sort restated as a stable lexsort on (sample, pool1 voxel row, voxel column, y inside the voxel,
    x inside the voxel, arrival index) of the clamped (x, y, sample).  The voxel of a pixel comes from geom.levels[0].cellx /
    celly and vx0 / vy0, not from the key tables the kernels read; the keys only size the start table, and the model asserts
    that they are non-decreasing along its order.  Returns start, perm, ti = (t, arrival index), xyb, feat_s and the
    time-order flag: set unless the clamped samples come as ascending contiguous runs in arrival order, each time-sorted
    (an event whose predecessor in arrival order has a larger clamped sample, or the same one and a larger t);
  * ref_export: the reference's edge_index from a column-major ELL (slot q of sorted position p at [q][p], slot 15 = degree):
    per destination in arrival order the self loop, then slots 0..deg-1 as ti[src].y.  A row is written only when its end
    is <= cap;
  * RingModel: the control block of dagr_stream_push / dagr_stream_push_multi word by word (include/dagr_b200.h, streaming
    blocks), the literal eviction search on the ring's t values, the clamped chunk size and stage offset, and the appended
    slots.  windows() gives the compact stream-major live order that dagr_graph_sort_ring[s] read;
  * ref_prepare: dagr_prepare_events / dagr_denormalize_pos in numpy float32 -- a rounded multiply, a rounded add of
    fl32(1e-3), truncation toward zero -- on inputs at the truncation edges (prepare_edges).

The last tests check the refusal of geometries whose B * ny1 * nx1 * CP sort keys do not fit the sort's 32-bit key.
"""
import ctypes as C

import numpy as np
import pytest
import torch

E_ARG, E_UNSUPPORTED = -1, -3
BAD = C.c_void_p(256)          # never dereferenced: the refused calls return before any CUDA call
CTL = 8                        # DAGR_RING_CTL


# ------------------------------------------------------------------------------------------------------------------------
# plain sort
# ------------------------------------------------------------------------------------------------------------------------
def clamp_xyb(geom, batch, pos):
    """the kernels' clamping of out-of-range events into the grid: int64 (x, y, sample)"""
    pos = np.asarray(pos, np.int64).reshape(-1, 3)
    x = np.clip(pos[:, 0], 0, geom.W - 1)
    y = np.clip(pos[:, 1], 0, geom.H - 1)
    b = np.clip(np.asarray(batch, np.int64), 0, geom.B - 1)
    return x, y, b


def ref_sort(geom, batch, pos, feat):
    """dict of start int64[NK + 1], perm int32[N], ti int32[N, 2], xyb uint32[N], feat_s float32[N], flag bool"""
    batch = np.asarray(batch, np.int64)
    pos = np.asarray(pos, np.int64).reshape(-1, 3)
    feat = np.asarray(feat, np.float32)
    N = len(batch)
    x, y, b = clamp_xyb(geom, batch, pos)
    lv = geom.levels[0]
    cx, cy = lv.cellx.numpy().astype(np.int64)[x], lv.celly.numpy().astype(np.int64)[y]
    xi, yi = x - geom.vx0.numpy()[cx], y - geom.vy0.numpy()[cy]
    arrival = np.arange(N)
    order = np.lexsort((arrival, xi, yi, cx, cy, b))
    key = b * (geom.ny1 * geom.nx1 * geom.CP) + geom.ykey.numpy()[y] + geom.xkey.numpy()[x]
    ks = key[order]
    assert np.all(np.diff(ks) >= 0), "the geometry's key order differs from the model's lexsort order"
    start = np.zeros(geom.NK + 1, np.int64)
    start[1:] = np.cumsum(np.bincount(key, minlength=geom.NK))
    assert np.all(start[ks] <= arrival) and np.all(arrival < start[ks + 1]), "start does not bound a key's run"
    t = pos[:, 2]
    flag = bool(N > 1 and np.any((b[:-1] > b[1:]) | ((b[:-1] == b[1:]) & (t[:-1] > t[1:]))))
    return dict(start=start, perm=order.astype(np.int32), ti=np.stack([t[order], order], 1).astype(np.int32),
                xyb=(x | y << 12 | b << 24)[order].astype(np.uint32), feat_s=feat[order], flag=flag)


def make_events(W, H, samples, n, seed, interleave=False, T=1_000_000):
    """batch int32[N], pos int32[N, 3], feat float32[N]: n uniform events per listed sample, time-sorted within each sample;
    samples one after the other in arrival order, or randomly interleaved (each sample's events keep their time order)"""
    rng = np.random.default_rng(seed)
    b = np.repeat(np.asarray(samples, np.int64), n)
    x, y = rng.integers(0, W, len(b)), rng.integers(0, H, len(b))
    t = np.concatenate([np.sort(rng.integers(0, T, n)) for _ in samples]) if len(b) else np.zeros(0, np.int64)
    if interleave:
        o = np.argsort(rng.random(len(b)), kind="stable")
        slot = np.empty(len(b), np.int64)
        for s in np.unique(b):                      # the k-th arrival of sample s takes its k-th event in time
            slot[np.flatnonzero(b[o] == s)] = np.flatnonzero(b == s)
        b, x, y, t = b[slot], x[slot], y[slot], t[slot]
    feat = rng.choice(np.array([-1.0, 1.0], np.float32), len(b))
    return b.astype(np.int32), np.stack([x, y, t], 1).astype(np.int32), feat


# ------------------------------------------------------------------------------------------------------------------------
# export
# ------------------------------------------------------------------------------------------------------------------------
def ref_export(perm, ti, nbr, cap=None):
    """(rowptr int64[N + 1], src int64[E], dst int64[E], fits bool[N]) from perm[N], ti [N, 2] and the ELL nbr [16, N]"""
    perm = np.asarray(perm, np.int64)
    ti = np.asarray(ti, np.int64).reshape(-1, 2)
    nbr = np.asarray(nbr, np.int64).reshape(16, -1)
    N = len(perm)
    inv = np.empty(N, np.int64)
    inv[perm] = np.arange(N)
    deg = nbr[15, inv]
    rowptr = np.zeros(N + 1, np.int64)
    rowptr[1:] = np.cumsum(deg + 1)
    dst = np.repeat(np.arange(N), deg + 1)
    q = np.arange(len(dst)) - rowptr[dst] - 1                   # -1: the self loop
    src = dst.copy()
    e = q >= 0
    src[e] = ti[nbr[q[e], inv[dst[e]]], 1]
    fits = rowptr[1:] <= (rowptr[N] if cap is None else cap)
    return rowptr, src, dst, fits


def ell_from_edges(edge_index, perm, N):
    """the ELL [16, N] whose export is edge_index: edges (arrival ids, dst ascending, self loop first) at the sorted positions
    of perm, slots in edge order"""
    src, dst = (np.asarray(v, np.int64) for v in edge_index)
    pos_of = np.empty(N, np.int64)
    pos_of[np.asarray(perm, np.int64)] = np.arange(N)
    m = src != dst
    src, dst = src[m], dst[m]
    first = np.zeros(N + 1, np.int64)
    first[1:] = np.cumsum(np.bincount(dst, minlength=N))
    nbr = np.full((16, N), -1, np.int64)
    nbr[np.arange(len(dst)) - first[dst], pos_of[dst]] = pos_of[src]
    nbr[15, pos_of] = first[1:] - first[:-1]
    return nbr


# ------------------------------------------------------------------------------------------------------------------------
# streaming rings
# ------------------------------------------------------------------------------------------------------------------------
SENT_I = -0x5a5a5a5b           # ring words the model has not written
SENT_F = np.float32(-777.25)


class RingModel:
    """S rings of `capacity` slots and their control block, as dagr_stream_push (single=True: one i32[8] block, batch =
    `sample`) or dagr_stream_push_multi (i32[S+1][8], batch = s) leave them"""

    def __init__(self, S, capacity, max_chunk, single=False, sample=0):
        assert capacity & (capacity - 1) == 0 and 1 <= max_chunk <= capacity and (S == 1 or not single)
        self.S, self.cap, self.mask, self.mc, self.single, self.sample = S, capacity, capacity - 1, max_chunk, single, sample
        self.ctl = np.zeros(CTL if single else CTL * (S + 1), np.int32)
        self.batch = np.full(S * capacity, SENT_I, np.int32)
        self.pos = np.full((S * capacity, 3), SENT_I, np.int32)
        self.feat = np.full(S * capacity, SENT_F, np.float32)

    def stage(self, hdr, events=()):
        """int32[4 S + 4 S max_chunk]: hdr = S rows {n_new, t_cut, event offset, word 3}; events = (x, y, t, p) rows placed
        from event 0 on; the rest of the event area holds a sentinel"""
        st = np.full(4 * self.S + 4 * self.S * self.mc, SENT_I, np.int32)
        st[:4 * self.S] = np.asarray(hdr, np.int64).reshape(-1)
        ev = np.asarray(events, np.int64).reshape(-1, 4)
        st[4 * self.S:4 * self.S + ev.size] = ev.reshape(-1)
        return st

    def reset(self, s):
        self.ctl[CTL * s:CTL * (s + 1)] = 0

    def push(self, stage):
        """one push; returns the streams whose chunk did not fit (the oldest events were dropped beyond t_cut)"""
        S, cap, mask, mc = self.S, self.cap, self.mask, self.mc
        hdr = np.asarray(stage[:4 * S], np.int64).reshape(S, 4)
        ev = np.asarray(stage[4 * S:4 * S + 4 * S * mc], np.int64).reshape(S * mc, 4)
        live, spilled = [], []
        for s in range(S):
            c = self.ctl[CTL * s:CTL * (s + 1)]
            head, n = int(c[0]), int(c[1])
            n_new, t_cut = min(max(int(hdr[s, 0]), 0), mc), int(hdr[s, 1])
            lo, hi = 0, n
            while lo < hi:                                            # first live event with t >= t_cut
                mid = (lo + hi) >> 1
                if self.pos[s * cap + ((head + mid) & mask), 2] < t_cut:
                    lo = mid + 1
                else:
                    hi = mid
            shift = lo
            if n - shift + n_new > cap:                               # the chunk does not fit: drop the oldest events
                shift = n + n_new - cap
                c[4] = 1
                spilled.append(s)
            c[0], c[5], c[1], c[2], c[3] = (head + shift) & mask, n - shift, n - shift + n_new, shift, n_new
            live.append(int(c[1]))
        off = np.concatenate([[0], np.cumsum(live)[:-1]])
        for s in range(S):
            self.ctl[CTL * s + 6] = off[s]
        if not self.single:
            self.ctl[CTL * S] = sum(live)
        for s in range(S):
            c = self.ctl[CTL * s:CTL * (s + 1)]
            n_new = int(c[3])
            eo = min(max(int(hdr[s, 2]), 0), S * mc - n_new)
            slot = s * cap + ((int(c[0]) + int(c[5]) + np.arange(n_new)) & mask)
            e = ev[eo:eo + n_new]
            self.pos[slot] = e[:, :3]
            self.feat[slot] = e[:, 3].astype(np.float32)
            self.batch[slot] = self.sample if self.single else s
        return spilled

    @property
    def total(self):
        return int(self.ctl[1]) if self.single else int(self.ctl[CTL * self.S])

    def slots(self):
        """ring slots of the live events in the compact stream-major order c < total"""
        out = [s * self.cap + ((int(self.ctl[CTL * s]) + np.arange(int(self.ctl[CTL * s + 1]))) & self.mask) for s in range(self.S)]
        return np.concatenate(out).astype(np.int64)

    def windows(self):
        """(batch, pos, feat) of the live events in the compact order: the inputs of ref_sort for the ring sorts"""
        sl = self.slots()
        return self.batch[sl], self.pos[sl], self.feat[sl]


# ------------------------------------------------------------------------------------------------------------------------
# input conversion
# ------------------------------------------------------------------------------------------------------------------------
def ref_prepare(pos, batch, x, ldx, W, H, T):
    """(pos_i int32[N, 3], batch_i int32[N], feat float32[N]): fl32(fl32(s * pos) + fl32(1e-3)) truncated toward zero, batch
    cast to int32 (two's complement wrap, as torch's .int()), feat = x[:, 0] of the [N, ldx] rows"""
    pos = np.asarray(pos, np.float32).reshape(-1, 3)
    s = np.array([W, H, T], np.float32)
    v = (pos * s).astype(np.float32) + np.float32(1e-3)
    assert v.dtype == np.float32
    pos_i = np.trunc(v).astype(np.int32)
    batch_i = np.asarray(batch, np.int64).astype(np.int32)
    feat = np.asarray(x, np.float32).reshape(-1, ldx)[:, 0]
    return pos_i, batch_i, feat


def fma_trunc(pos, s):
    """what a fused multiply-add would give: the exact product plus fl32(1e-3), rounded once to fp32, truncated.  The float64
    sum is exact: a 48-bit product of values < 2^13 and fl32(1e-3) >= 2^-10 span fewer than 53 bits"""
    exact = np.asarray(pos, np.float32).astype(np.float64) * float(s) + float(np.float32(1e-3))
    return np.trunc(exact.astype(np.float32)).astype(np.int32)


def prepare_edges(s, ulps=8):
    """fp32 inputs at the truncation edges of one axis of scale s: for every integer k in [0, s], fl32(k / s) and its two fp32
    neighbours, and the inputs within `ulps` fp32 steps of fl32((k - 1e-3) / s) whose fl32(s * pos) lies within 2e-3 of an
    integer.  The margin past 1e-3 keeps the products just more than 1e-3 below an integer, where the rounding of the add
    decides the truncation and a fused multiply-add gives another integer"""
    k = np.arange(s + 1, dtype=np.float64)
    base = (k / s).astype(np.float32)
    near = ((k - 1e-3) / s).astype(np.float32)
    cand = [near]
    up, dn = near, near
    for _ in range(ulps):
        up, dn = np.nextafter(up, np.float32(2)), np.nextafter(dn, np.float32(-1))
        cand += [up, dn]
    cand = np.concatenate(cand)
    prod = (cand * np.float32(s)).astype(np.float64)
    cand = cand[np.abs(prod - np.round(prod)) <= 2e-3]
    out = np.concatenate([base, np.nextafter(base, np.float32(2)), np.nextafter(base, np.float32(-1)), cand])
    return np.unique(out[out >= 0])


def edge_rows(W, H, T):
    """pos float32 [N, 3]: the edge inputs of the three axes, each column cycled to the longest"""
    cols = [prepare_edges(W), prepare_edges(H), prepare_edges(T)]
    n = max(len(c) for c in cols)
    return np.stack([np.resize(c, n) for c in cols], 1)


# ------------------------------------------------------------------------------------------------------------------------
# tests: models
# ------------------------------------------------------------------------------------------------------------------------
def _geom(W, H, B, radius=0.01):
    from dagr_b200.geometry import Geometry
    return Geometry(W, H, B, radius=radius, device="cpu")


def test_ref_sort_on_a_hand_sorted_stream():
    """240 x 180 (pool1 voxel columns and rows start at 0, 5, 9): voxel-major, then y, x inside the voxel, then arrival"""
    geom = _geom(240, 180, 2)
    assert geom.vx0[:3].tolist() == [0, 5, 9] and geom.vy0[:3].tolist() == [0, 5, 9]
    #                 x    y    t
    ev = np.array([[6, 0, 50],          # 0: sample 1, voxel (1, 0)
                   [7, 1, 10],          # 1: sample 0, voxel (1, 0), y 1
                   [8, 0, 20],          # 2: sample 0, voxel (1, 0), y 0
                   [0, 7, 30],          # 3: sample 0, voxel (0, 1)
                   [8, 0, 40],          # 4: sample 0, same pixel as 2, later
                   [4, 4, 35]])         # 5: sample 0, voxel (0, 0), earlier than event 4
    batch = np.array([1, 0, 0, 0, 0, 0])
    r = ref_sort(geom, batch, ev, np.arange(6, dtype=np.float32))
    assert r["perm"].tolist() == [5, 2, 4, 1, 3, 0]
    assert r["ti"][:, 0].tolist() == [35, 20, 40, 10, 30, 50] and r["ti"][:, 1].tolist() == r["perm"].tolist()
    assert r["xyb"][0] == 4 | 4 << 12 and r["xyb"][5] == 6 | 1 << 24
    assert r["feat_s"].tolist() == [5, 2, 4, 1, 3, 0]
    assert r["start"][-1] == 6 and r["start"][geom.NK // 2] == 5
    assert r["flag"]                                   # event 5 (t = 35) arrives after event 4 (t = 40) of its sample
    ev[5, 2] = 40
    assert ref_sort(geom, batch, ev, np.zeros(6, np.float32))["flag"]            # sample 1 still arrives before sample 0
    assert not ref_sort(geom, batch[1:], ev[1:], np.zeros(5, np.float32))["flag"]


def test_ref_sort_flag_rules_and_clamping():
    geom = _geom(240, 180, 3)
    pos = np.array([[1, 1, 10], [2, 2, 10], [3, 3, 5], [-1, 180, 7], [240, -5, 8], [10 ** 6, 10 ** 6, 9]])
    # equal times and a drop into the next sample leave the flag clear; the samples compared are the clamped ones (3 and
    # 2^20 are sample 2 at B = 3, so the times 7, 8, 9 must ascend)
    assert not ref_sort(geom, [0, 0, 1, 2, 3, 1 << 20], pos, np.zeros(6))["flag"]
    assert ref_sort(geom, [0, 0, 0, 2, 3, 1 << 20], pos, np.zeros(6))["flag"]
    pos[4, 2] = 6
    assert ref_sort(geom, [0, 0, 1, 2, 3, 1 << 20], pos, np.zeros(6))["flag"]      # 7 -> 6 inside the clamped sample 2
    x, y, b = clamp_xyb(geom, [-1, 3, 1 << 20, 0, 0, 0], pos)
    assert x.tolist() == [1, 2, 3, 0, 239, 239] and y.tolist() == [1, 2, 3, 179, 0, 179] and b.tolist() == [0, 2, 2, 0, 0, 0]


@pytest.mark.parametrize("wh,B,radius", [((240, 180), 3, 0.01), ((640, 480), 8, 0.01), ((1280, 720), 2, 12.5 / 1280)])
def test_ref_sort_and_ref_export_reproduce_the_graph_oracle(wh, B, radius):
    """ELL from the oracle's edges at ref_sort's positions -> ref_export gives the oracle's edge_index back: ties the sort model
    to graph_oracle.c"""
    from tests.test_l1_kernels_cpu import oracle_edges
    geom = _geom(*wh, B, radius)
    batch, pos, feat = make_events(wh[0] // 4, wh[1] // 4, range(B), 3000, seed=B, T=20_000)     # dense: most nodes have edges
    r = ref_sort(geom, batch, pos, feat)
    edges = oracle_edges(geom, torch.from_numpy(batch), torch.from_numpy(pos)).numpy()
    nbr = ell_from_edges(edges, r["perm"], len(batch))
    rowptr, src, dst, fits = ref_export(r["perm"], r["ti"], nbr)
    assert np.array_equal(np.stack([src, dst]), edges) and fits.all() and rowptr[-1] == edges.shape[1]
    assert (nbr[15] > 0).mean() > 0.8 and nbr[15].max() == 15


def test_ref_export_cap_keeps_whole_rows_only():
    perm = np.array([2, 0, 1])
    ti = np.array([[0, 7], [0, 8], [0, 9]])
    nbr = np.full((16, 3), -1)
    nbr[15] = [1, 2, 0]                                # degrees at sorted positions 0, 1, 2 (arrival 2, 0, 1)
    nbr[0, 0], nbr[0, 1], nbr[1, 1] = 1, 2, 0
    rowptr, src, dst, fits = ref_export(perm, ti, nbr, cap=5)
    assert rowptr.tolist() == [0, 3, 4, 6]
    assert src.tolist() == [0, 9, 7, 1, 2, 8] and dst.tolist() == [0, 0, 0, 1, 2, 2]
    assert fits.tolist() == [True, True, False]


def test_make_events_interleaves_without_breaking_time_order():
    b, pos, _ = make_events(240, 180, [0, 1, 5], 200, seed=3, interleave=True)
    assert len(np.unique(b[:30])) == 3
    for s in (0, 1, 5):
        assert np.all(np.diff(pos[b == s, 2]) >= 0)


def test_ring_model_known_answer_at_capacity_8():
    """two streams of 8 slots: a wrap, an overflow with an eviction in the other stream, then a reset of block 0 alone"""
    m = RingModel(2, 8, 8)
    ev = lambda ts, p=1: [[i, i + 1, t, p] for i, t in enumerate(ts)]          # noqa: E731
    m.push(m.stage([[6, 0, 0, 0], [3, 0, 6, 0]], ev(range(10, 16)) + ev([100, 101, 102], -1)))
    assert m.ctl.reshape(3, 8).tolist() == [[0, 6, 0, 6, 0, 0, 0, 0], [0, 3, 0, 3, 0, 0, 6, 0], [9, 0, 0, 0, 0, 0, 0, 0]]
    assert m.batch[8:11].tolist() == [1, 1, 1] and m.feat[8] == -1 and m.pos[9].tolist() == [1, 2, 101]
    m.push(m.stage([[4, 13, 0, 77], [0, 0, 0, -5]], ev(range(16, 20))))         # word 3 is ignored
    assert m.ctl.reshape(3, 8).tolist() == [[3, 7, 3, 4, 0, 3, 0, 0], [0, 3, 0, 0, 0, 3, 7, 0], [10, 0, 0, 0, 0, 0, 0, 0]]
    assert m.pos[[6, 7, 0, 1], 2].tolist() == [16, 17, 18, 19]                  # the chunk wraps the ring's end
    assert m.push(m.stage([[3, 0, 0, 0], [0, 101, 0, 0]], ev(range(20, 23)))) == [0]
    assert m.ctl.reshape(3, 8).tolist() == [[5, 8, 2, 3, 1, 5, 0, 0], [1, 2, 1, 0, 0, 2, 8, 0], [10, 0, 0, 0, 0, 0, 0, 0]]
    assert m.windows()[1][:, 2].tolist() == [15, 16, 17, 18, 19, 20, 21, 22, 101, 102]
    m.reset(0)
    assert m.push(m.stage([[2, 0, 1, 0], [1, 0, 0, 0]], ev([103, 5, 6]))) == []  # stream 0 reads events 1, 2; stream 1 event 0
    assert m.ctl.reshape(3, 8).tolist() == [[0, 2, 0, 2, 0, 0, 0, 0], [1, 3, 0, 1, 0, 2, 2, 0], [5, 0, 0, 0, 0, 0, 0, 0]]
    b, p, f = m.windows()
    assert b.tolist() == [0, 0, 1, 1, 1] and p[:, 2].tolist() == [5, 6, 101, 102, 103]
    assert m.pos[7, 2] == 17                           # the evicted slot before stream 0's first live event keeps a larger t
    assert m.slots().tolist() == [0, 1, 9, 10, 11]


def test_ring_model_clamps_the_chunk_and_the_stage_offset():
    m = RingModel(2, 8, 4)
    m.push(m.stage([[9, 0, 6, 0], [-3, 0, 0, 0]], [[k, k, 100 + k, 1] for k in range(8)]))
    # n_new 9 -> 4, its offset 6 -> 2 * 4 - 4 = 4; stream 1 appends nothing
    assert m.ctl.reshape(3, 8)[:2, :4].tolist() == [[0, 4, 0, 4], [0, 0, 0, 0]]
    assert m.pos[:4, 2].tolist() == [104, 105, 106, 107] and (m.pos[4:, 2] == SENT_I).all()
    single = RingModel(1, 4, 4, single=True, sample=3)
    single.push(single.stage([[4, 0, 0, 0]], [[1, 1, t, -1] for t in range(4)]))
    single.push(single.stage([[4, 2, -9, 0]], [[1, 1, t, -1] for t in range(10, 14)]))
    # t_cut = 2 evicts 2, the chunk of 4 then overflows: 2 more are dropped
    assert single.ctl.tolist() == [0, 4, 4, 4, 1, 0, 0, 0] and single.total == 4
    assert single.windows()[0].tolist() == [3] * 4 and single.windows()[1][:, 2].tolist() == [10, 11, 12, 13]


def test_ref_prepare_equals_the_oracle_on_the_truncation_edges():
    from oracle.ref_ops import denormalize_pos
    for W, H in ((640, 480), (1280, 720)):
        T = 1_000_000
        pos = edge_rows(W, H, T)
        got = ref_prepare(pos, np.zeros(len(pos)), np.zeros((len(pos), 1)), 1, W, H, T)[0]
        ref = denormalize_pos(torch.from_numpy(pos), W, H, T).numpy()
        assert np.array_equal(got, ref), (W, H)
        # the set holds inputs where a fused multiply-add truncates to another integer, on both sensor axes
        for d, s in enumerate((W, H)):
            assert (fma_trunc(pos[:, d], s) != got[:, d]).sum() >= 4, (W, H, d)
        # and inputs where the 1e-3 decides: fl(s pos) just below an integer, lifted to it
        prod = (pos[:, 0] * np.float32(W)).astype(np.float32)
        assert ((np.trunc(prod) != got[:, 0]) & (prod > 0)).sum() > W // 2


def test_ref_prepare_batch_cast_and_row_stride():
    pos = np.zeros((3, 3), np.float32)
    x = np.arange(9, dtype=np.float32).reshape(3, 3)
    _, b, f = ref_prepare(pos, [(1 << 32) + 5, -1, 1 << 31], x, 3, 4, 4, 4)
    assert b.tolist() == [5, -1, -(1 << 31)] and f.tolist() == [0, 3, 6]


# ------------------------------------------------------------------------------------------------------------------------
# tests: 32-bit sort keys
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H,B", [(4096, 4096, 128), (4096, 4096, 127), (3840, 2160, 255), (4096, 4096, 255)])
def test_geometry_refuses_sort_keys_past_31_bits(W, H, B):
    from dagr_b200.geometry import Geometry
    with pytest.raises(ValueError, match="32-bit sort key"):
        Geometry(W, H, B, radius=0.003, device="cpu")


def _overflowing(B):
    """a c_geom whose B * ny1 * nx1 * CP >= 2^31, with NK as ctypes would have truncated it"""
    geom = _geom(4096, 4096, 1, 0.003)
    g = geom.c_geom
    g.B = B
    g.NK = B * geom.ny1 * geom.nx1 * geom.CP              # ctypes keeps the low 32 bits
    assert g.NK != B * geom.ny1 * geom.nx1 * geom.CP
    return geom, g


@pytest.mark.parametrize("B", [127, 255])
def test_check_config_refuses_sort_keys_past_31_bits(B):
    from dagr_b200 import _lib
    lib = _lib.load()
    geom, g = _overflowing(B)
    assert lib.dagr_check_config(C.byref(g), 10, 3, 16, b"relu") == E_UNSUPPORTED
    assert "32-bit sort key" in lib.dagr_last_error().decode()
    ok = _geom(4096, 4096, 1, 0.003)
    assert lib.dagr_check_config(C.byref(ok.c_geom), 10, 3, 16, b"relu") == 0
    ok.c_geom.NK += 1
    assert lib.dagr_check_config(C.byref(ok.c_geom), 10, 3, 16, b"relu") == E_UNSUPPORTED
    assert "NK" in lib.dagr_last_error().decode()


@pytest.mark.parametrize("entry", ["dagr_graph_sort", "dagr_graph_sort_ring", "dagr_graph_sort_rings"])
def test_graph_sorts_refuse_sort_keys_past_31_bits(entry):
    from dagr_b200 import _lib
    lib = _lib.load()
    geom, g = _overflowing(127)
    gp = C.byref(g)
    if entry == "dagr_graph_sort":
        rc = lib.dagr_graph_sort(gp, BAD, BAD, BAD, 10, BAD, BAD, BAD, BAD, BAD, BAD, BAD, BAD, BAD, None, None)
    elif entry == "dagr_graph_sort_ring":
        rc = lib.dagr_graph_sort_ring(gp, BAD, BAD, BAD, 1 << 10, BAD, BAD, BAD, BAD, BAD, BAD, BAD, BAD, BAD, BAD, None, None)
    else:
        rc = lib.dagr_graph_sort_rings(gp, BAD, BAD, BAD, 1 << 10, 127, BAD, BAD, BAD, BAD, BAD, BAD, BAD, BAD, BAD, BAD, None, None)
    assert rc == E_ARG
    assert "32-bit sort key" in lib.dagr_last_error().decode()
