"""csrc/graph.cu on its own, through the C-ABI, bit for bit against the numpy models of tests/test_graph_sort_cpu.py.

  * dagr_graph_sort: start[0..NK], perm, ti, xyb, feat_s (as bits) and the not-time-sorted flag equal ref_sort; count is zero
    again on exit and nothing is written past N.  Cases reach sample indices up to 254, x and y at 4095, clamped out-of-range
    x / y / batch values, a 5000-event pixel, N = 0 and 1, and the benchmark's 640 x 480 at B = 8;
  * dagr_graph_export: rowptr and the edge words against ref_export on a synthetic ELL, at N on either side of the scan's
    2048-element tile and of the 256-tile chunks of its block-sum pass, with cap = E, E - 1 and inside a row;
  * dagr_stream_push / dagr_stream_push_multi: scripted pushes against RingModel, the whole control block and every ring slot
    compared after each push (slots the model did not write keep their sentinel).  After each push dagr_graph_sort_ring[s]
    must equal ref_sort on the model's compact live windows;
  * dagr_prepare_events / dagr_denormalize_pos against ref_prepare on the truncation-edge inputs.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_graph_sort_cpu import CTL, RingModel, edge_rows, make_events, ref_export, ref_prepare, ref_sort

pytestmark = pytest.mark.gpu

SENT = -0x3c3c3c3d             # output words the kernels must not write


def _lib():
    from dagr_b200 import _lib as L
    return L, L.load()


def P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _geom(W, H, B, radius=0.01):
    from dagr_b200.geometry import Geometry
    return Geometry(W, H, B, radius=radius, device="cuda")


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).astype(np.int64).astype(np.int32)))


def _bits(a):
    """int32 view of float32 / uint32 data"""
    return torch.from_numpy(np.ascontiguousarray(a)).view(torch.int32) if isinstance(a, np.ndarray) else a.view(torch.int32)


# ------------------------------------------------------------------------------------------------------------------------
# the sort and its checks
# ------------------------------------------------------------------------------------------------------------------------
class SortBufs:
    """outputs (sentinel-filled) and work buffers of one sort over N slots"""

    def __init__(self, geom, N):
        L, lib = _lib()
        n = max(N, 1) + 1
        dev = "cuda"
        nb = int(lib.dagr_scan_blocks(max(geom.NK + 1, N + 1))) + 2
        self.key = torch.zeros(n, dtype=torch.int32, device=dev)
        self.tmp = torch.zeros(n, dtype=torch.int32, device=dev)
        self.count = torch.zeros(geom.NK + 1, dtype=torch.int32, device=dev)
        self.blocksums = torch.zeros(nb, dtype=torch.int32, device=dev)
        self.start = torch.full((geom.NK + 2,), SENT, dtype=torch.int32, device=dev)
        self.perm = torch.full((n,), SENT, dtype=torch.int32, device=dev)
        self.ti = torch.full((n, 2), SENT, dtype=torch.int32, device=dev)
        self.xyb = torch.full((n,), SENT, dtype=torch.int32, device=dev)
        self.feat_s = torch.full((n,), SENT, dtype=torch.int32, device=dev)
        self.flags = torch.zeros(1, dtype=torch.int32, device=dev)

    def reset(self):
        for t in (self.start, self.perm, self.ti, self.xyb, self.feat_s):
            t.fill_(SENT)
        self.flags.zero_()

    def args(self):
        return [P(self.key), P(self.tmp), P(self.count), P(self.blocksums), P(self.start), P(self.perm), P(self.ti), P(self.xyb),
                P(self.feat_s), P(self.flags), st()]


def check_sort(geom, bufs, ref, total, what):
    """the sort's outputs equal the model at the positions below `total`; nothing is written at or past it, count is zero"""
    torch.cuda.synchronize()
    NK = geom.NK
    assert torch.equal(bufs.start[:NK + 1].cpu(), _i32(ref["start"])), f"{what}: start"
    assert int(bufs.start[NK + 1]) == SENT, f"{what}: start written past NK"
    assert int(bufs.count.abs().sum()) == 0, f"{what}: count is not zero again on exit"
    assert torch.equal(bufs.perm[:total].cpu(), _i32(ref["perm"])), f"{what}: perm"
    assert torch.equal(bufs.ti[:total].cpu(), _i32(ref["ti"])), f"{what}: ti"
    assert torch.equal(bufs.xyb[:total].cpu(), _bits(ref["xyb"])), f"{what}: xyb"
    assert torch.equal(bufs.feat_s[:total].cpu(), _bits(np.asarray(ref["feat_s"], np.float32))), f"{what}: feat_s"
    for name in ("perm", "ti", "xyb", "feat_s"):
        assert bool((getattr(bufs, name)[total:] == SENT).all()), f"{what}: {name} written at or past the total"
    assert int(bufs.flags[0]) == int(ref["flag"]), f"{what}: flag {int(bufs.flags[0])}, model {ref['flag']}"


def plain_sort(geom, batch, pos, feat):
    L, lib = _lib()
    N = len(batch)
    bufs = SortBufs(geom, N)
    inp = [_i32(batch).cuda(), _i32(pos).cuda(), torch.from_numpy(np.asarray(feat, np.float32)).cuda()]
    if N == 0:
        inp = [torch.zeros(4, dtype=t.dtype, device="cuda") for t in inp]
    L.check(lib.dagr_graph_sort(C.byref(geom.c_geom), *map(P, inp), N, *bufs.args()), "sort")
    return bufs


def _evs(W, H, samples, n, seed, **kw):
    return lambda: make_events(W, H, samples, n, seed, **kw)


def _corners(seed):
    b, pos, f = make_events(4096, 4096, [0], 60000, seed)
    pos[:8, :2] = [[4095, 4095], [4095, 0], [0, 4095], [4095, 4095], [4095, 4094], [4094, 4095], [0, 0], [2048, 4095]]
    return b, pos, f


def _out_of_range(seed):
    """240 x 180 at B = 3: x, y and batch values of -1, W / H / B and 2^20 mixed into valid events"""
    b, pos, f = make_events(240, 180, [0, 1, 2], 3000, seed, interleave=True)
    rng = np.random.default_rng(seed)
    k = rng.choice(len(b), 600, replace=False)
    pos[k[:100], 0] = -1; pos[k[100:200], 0] = 240; pos[k[200:250], 0] = 1 << 20
    pos[k[250:350], 1] = -1; pos[k[350:450], 1] = 180; pos[k[450:500], 1] = 1 << 20
    b[k[500:540]] = -1; b[k[540:580]] = 3; b[k[580:]] = 1 << 20
    return b, pos, f


def _hot_pixel(seed):
    """640 x 480 at B = 2: 5000 events on one pixel of sample 1 between background events"""
    b, pos, f = make_events(640, 480, [0, 1], 20000, seed)
    rng = np.random.default_rng(seed)
    k = np.sort(rng.choice(np.flatnonzero(b == 1), 5000, replace=False))
    pos[k, 0], pos[k, 1] = 321, 239
    return b, pos, f


PLAIN = {
    "240x180-B1-samples-up-to-254-clamped-to-0": (dict(W=240, H=180, B=1), _evs(240, 180, [0, 1, 127, 128, 254], 2000, 1)),
    "240x180-B255-samples-0-1-127-128-254": (dict(W=240, H=180, B=255), _evs(240, 180, [0, 1, 127, 128, 254], 2000, 2)),
    "640x480-B8-interleaved-bench-shape": (dict(W=640, H=480, B=8), _evs(640, 480, range(8), 25000, 3, interleave=True)),
    "1280x720-B2-r13": (dict(W=1280, H=720, B=2, radius=12.5 / 1280), _evs(1280, 720, [0, 1], 40000, 4)),
    "4096x4096-B1-x-y-4095": (dict(W=4096, H=4096, B=1, radius=0.003), lambda: _corners(5)),
    "240x180-B3-out-of-range-x-y-batch": (dict(W=240, H=180, B=3), lambda: _out_of_range(6)),
    "640x480-B2-hot-pixel-5000": (dict(W=640, H=480, B=2), lambda: _hot_pixel(7)),
    "240x180-N0": (dict(W=240, H=180, B=2), _evs(240, 180, [], 0, 8)),
    "240x180-N1": (dict(W=240, H=180, B=2), _evs(240, 180, [1], 1, 9)),
}


@pytest.mark.parametrize("name", list(PLAIN))
def test_plain_sort_equals_the_model(name):
    gk, mk = PLAIN[name]
    geom = _geom(gk["W"], gk["H"], gk["B"], gk.get("radius", 0.01))
    batch, pos, feat = mk()
    ref = ref_sort(geom, batch, pos, feat)
    bufs = plain_sort(geom, batch, pos, feat)
    check_sort(geom, bufs, ref, len(batch), name)
    if name.startswith("4096"):
        assert (ref["xyb"] & 0xfff).max() == 4095 and ((ref["xyb"] >> 12) & 0xfff).max() == 4095
    if "254" in name:
        assert (ref["xyb"] >> 24).max() == (254 if "B255" in name else 0)
    if "hot-pixel" in name:                                         # the pixel's bin, in arrival order
        p = np.flatnonzero(ref["xyb"] == (321 | 239 << 12 | 1 << 24))
        assert len(p) >= 5000 and np.all(np.diff(ref["perm"][p]) > 0) and np.ptp(p) == len(p) - 1


@pytest.mark.parametrize("case,flag", [("inversion-inside-a-sample", 1), ("equal-times", 0), ("drop-across-samples", 0),
                                       ("drop-across-interleaved-samples", 1)])
def test_plain_sort_time_order_flag(case, flag):
    geom = _geom(240, 180, 2)
    batch, pos, feat = make_events(240, 180, [0, 1], 3000, 11, interleave="interleaved" in case)
    if case == "inversion-inside-a-sample":
        i = [j for j in np.flatnonzero(batch == 1)[1000:] if batch[j - 1] == 1 and pos[j - 1, 2] > 0][0]
        pos[i, 2] = pos[i - 1, 2] - 1
    elif case == "equal-times":
        pos[:, 2] = 7
    else:
        assert np.any((batch[1:] != batch[:-1]) & (pos[:-1, 2] > pos[1:, 2]))
    ref = ref_sort(geom, batch, pos, feat)
    assert ref["flag"] == bool(flag)
    check_sort(geom, plain_sort(geom, batch, pos, feat), ref, len(batch), case)


# ------------------------------------------------------------------------------------------------------------------------
# export
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 2047, 2048, 2049, 524288, 524289, 526337])
def test_export_equals_the_model_around_the_scan_tiles(N):
    L, lib = _lib()
    rng = np.random.default_rng(N)
    perm = rng.permutation(N)
    ti = np.stack([rng.integers(-(1 << 31), 1 << 31, N), rng.integers(0, 1 << 31, N)], 1)
    nbr = rng.integers(0, N, (16, N))
    nbr[15] = rng.integers(0, 16, N)
    rowptr_ref, src, dst, _ = ref_export(perm, ti, nbr)
    E = int(rowptr_ref[N])
    caps = {"E": E, "E-1": E - 1}
    deg = np.diff(rowptr_ref) - 1                                   # per destination, arrival order
    rows = np.flatnonzero(deg >= 2)
    if len(rows):
        mid = int(rows[len(rows) // 2])
        caps["inside-a-row"] = int(rowptr_ref[mid]) + 2
    d_perm, d_ti, d_nbr = _i32(perm).cuda(), _i32(ti).cuda(), _i32(nbr).cuda()
    nb = int(lib.dagr_scan_blocks(N + 1)) + 2
    if N > 2048 * 256:
        assert int(lib.dagr_scan_blocks(N)) > 256                   # the block sums take a second 256-tile chunk
    for what, cap in caps.items():
        inv = torch.zeros(N, dtype=torch.int32, device="cuda")
        rowptr = torch.full((N + 2,), SENT, dtype=torch.int32, device="cuda")
        blocksums = torch.zeros(nb, dtype=torch.int32, device="cuda")
        es = torch.full((E + 64,), SENT, dtype=torch.int64, device="cuda")
        ed = torch.full((E + 64,), SENT, dtype=torch.int64, device="cuda")
        L.check(lib.dagr_graph_export(None, N, P(d_perm), P(d_ti), P(d_nbr), P(inv), P(rowptr), P(blocksums), P(es), P(ed), cap,
                                      st()), "export")
        torch.cuda.synchronize()
        _, _, _, fits = ref_export(perm, ti, nbr, cap)
        assert torch.equal(rowptr[:N + 1].cpu(), _i32(rowptr_ref)), (N, what)
        assert int(rowptr[N + 1]) == SENT
        written = np.repeat(fits, np.diff(rowptr_ref) if N else 0)
        exp_s = np.where(written, src, SENT)
        exp_d = np.where(written, dst, SENT)
        assert torch.equal(es[:E].cpu(), torch.from_numpy(exp_s)), (N, what)
        assert torch.equal(ed[:E].cpu(), torch.from_numpy(exp_d)), (N, what)
        assert bool((es[E:] == SENT).all()) and bool((ed[E:] == SENT).all()), (N, what)
        if what == "E":
            assert fits.all()
        elif what == "E-1":
            assert fits[:-1].all() and not fits[-1]
        else:
            assert fits[:mid].all() and not fits[mid:].any()


# ------------------------------------------------------------------------------------------------------------------------
# streaming rings
# ------------------------------------------------------------------------------------------------------------------------
class DeviceRings:
    """the device side of a RingModel: the same sentinels in every slot, a zeroed control block, and the ring sort"""

    def __init__(self, m, geom):
        self.m, self.geom = m, geom
        self.ctl = torch.from_numpy(m.ctl.copy()).cuda()
        self.batch = torch.from_numpy(m.batch.copy()).cuda()
        self.pos = torch.from_numpy(m.pos.copy()).cuda()
        self.feat = torch.from_numpy(m.feat.copy()).cuda()
        self.stage = torch.zeros(4 * m.S + 4 * m.S * m.mc, dtype=torch.int32, device="cuda")
        self.sort = SortBufs(geom, m.S * m.cap)

    def push(self, stage):
        L, lib = _lib()
        m = self.m
        self.stage.copy_(torch.from_numpy(stage))
        if m.single:
            rc = lib.dagr_stream_push(P(self.ctl), P(self.stage), P(self.batch), P(self.pos), P(self.feat), m.cap, m.mc, m.sample, st())
        else:
            rc = lib.dagr_stream_push_multi(P(self.ctl), P(self.stage), P(self.batch), P(self.pos), P(self.feat), m.cap, m.S, m.mc, st())
        L.check(rc, "push")
        return m.push(stage)

    def reset(self, s):
        self.ctl[CTL * s:CTL * (s + 1)] = 0
        self.m.reset(s)

    def check_rings(self, what):
        torch.cuda.synchronize()
        m = self.m
        assert torch.equal(self.ctl.cpu(), torch.from_numpy(m.ctl)), f"{what}: ctl {self.ctl.cpu().view(-1, 8).tolist()[:4]} model {m.ctl.reshape(-1, 8).tolist()[:4]}"
        assert torch.equal(self.batch.cpu(), torch.from_numpy(m.batch)), f"{what}: batch"
        assert torch.equal(self.pos.cpu(), torch.from_numpy(m.pos)), f"{what}: pos"
        assert torch.equal(self.feat.cpu().view(torch.int32), torch.from_numpy(m.feat).view(torch.int32)), f"{what}: feat"

    def check_sort(self, what):
        L, lib = _lib()
        m, g, b = self.m, self.geom, self.sort
        b.reset()
        if m.single:
            rc = lib.dagr_graph_sort_ring(C.byref(g.c_geom), P(self.batch), P(self.pos), P(self.feat), m.cap, P(self.ctl), *b.args())
        else:
            rc = lib.dagr_graph_sort_rings(C.byref(g.c_geom), P(self.batch), P(self.pos), P(self.feat), m.cap, m.S, P(self.ctl),
                                           *b.args())
        L.check(rc, "ring sort")
        ref = ref_sort(g, *m.windows())
        check_sort(g, b, ref, m.total, what)
        return ref


def script(dev, steps, rng, reset_at=None, fill=True):
    """scripted pushes with every control path: per stream and step, t_cut at a live event's t, below the oldest, above the
    newest or between; n_new inside [0, max_chunk], 0, negative or above max_chunk; stream 1 of every 3 left empty for the
    first steps; one out-of-range event offset per step and garbage in word 3.  With `fill`, steps 2, 3, ... keep every live
    event and push max_chunk events per stream until the rings have overflowed.  Every push is compared with the model, ring
    slots and sort included.  Returns the control paths reached."""
    m = dev.m
    S, mc = m.S, m.mc
    fill_steps = range(2, 3 + m.cap // mc) if fill else ()
    last_t = rng.integers(0, 1000, S)
    seen = set()
    for k in range(steps):
        if k == reset_at:
            live = m.ctl.reshape(-1, CTL)[:S, 1]
            s = S // 2 if live[S // 2] > 0 or not live.any() else int(np.flatnonzero(live)[0])
            seen.add("reset" if live[s] > 0 else "reset-empty")
            dev.reset(s)
            last_t[s] = 0                                               # the stream restarts at an earlier time
        hdr, events, o = [], [], 0
        for s in range(S):
            c = m.ctl[CTL * s:CTL * (s + 1)]
            head, n = int(c[0]), int(c[1])
            live_t = m.pos[s * m.cap + ((head + np.arange(n)) & m.mask), 2]
            mode = 1 if k in fill_steps else (k + s) % 4
            if mode == 0 and n:
                t_cut = int(live_t[rng.integers(0, n)]); seen.add("t_cut-at-a-live-t")
            elif mode == 1:
                t_cut = int(live_t[0]) - 5 if n else -5; seen.add("t_cut-below-oldest")
            elif mode == 2:
                t_cut = int(last_t[s]) + 1; seen.add("t_cut-above-newest")
            else:
                t_cut = int(last_t[s]) - int(rng.integers(0, 3000))
            nm = (2 * k + s) % 5
            if k < 3 and s % 3 == 1 and S >= 3:
                n_new = 0
            elif k in fill_steps:
                n_new = mc
            elif nm == 0:
                n_new = 0; seen.add("n_new-0")
            elif nm == 1:
                n_new = -int(rng.integers(1, 100)); seen.add("n_new-negative")
            elif nm == 2:
                n_new = mc + int(rng.integers(1, 100)); seen.add("n_new-above-max_chunk")
            else:
                n_new = int(rng.integers(1, mc + 1))
            cnt = min(max(n_new, 0), mc)
            if cnt == m.cap and n > 0:
                seen.add("chunk-of-capacity-into-non-empty")
            t = last_t[s] + np.cumsum(rng.integers(0, 40, cnt))
            if cnt:
                last_t[s] = t[-1]
            events += [np.stack([rng.integers(0, 240, cnt), rng.integers(0, 180, cnt), t, rng.choice([-1, 1], cnt)], 1)]
            off = o
            if s == k % S:
                off = [-3, S * mc + 17, (S * mc) // 2 + 1][k % 3]; seen.add("offset-out-of-range")
            hdr.append([n_new, t_cut, off, int(rng.integers(-(1 << 31), 1 << 31))])
            o += cnt
        sticky = np.flatnonzero(m.ctl.reshape(-1, CTL)[:S, 4] == 1)
        spilled = dev.push(m.stage(hdr, np.concatenate(events)))
        blocks = m.ctl.reshape(-1, CTL)[:S]
        if ((blocks[:, 0] + blocks[:, 1]) > m.cap).any():
            seen.add("window-wraps")
        if spilled:
            seen.add("overflow")
        if set(sticky) - set(spilled):
            seen.add("overflow-stays-set")
        live = blocks[:, 1]
        nz = np.flatnonzero(live > 0)
        if len(nz) >= 2 and (live[nz[0]:nz[-1]] == 0).any():
            seen.add("empty-streams-between")
        dev.check_rings(f"step {k}")
        dev.check_sort(f"sort after step {k}")
    return seen


COMMON = {"t_cut-at-a-live-t", "t_cut-below-oldest", "t_cut-above-newest", "n_new-0", "n_new-negative", "n_new-above-max_chunk",
          "offset-out-of-range", "overflow", "overflow-stays-set", "window-wraps", "reset"}

RINGS = {   # name: (S, capacity, max_chunk, single, steps, paths that must be reached besides COMMON)
    "single-cap64-chunk16": (1, 64, 16, True, 14, set()),
    "single-cap256-chunk=cap": (1, 256, 256, True, 12, {"chunk-of-capacity-into-non-empty"}),
    "S1-cap64-chunk=cap": (1, 64, 64, False, 12, {"chunk-of-capacity-into-non-empty"}),
    "S2-cap256-chunk96": (2, 256, 96, False, 16, set()),
    "S31-cap64-chunk=cap": (31, 64, 64, False, 12, {"chunk-of-capacity-into-non-empty", "empty-streams-between"}),
    "S32-cap256-chunk96": (32, 256, 96, False, 14, {"empty-streams-between"}),
    "S33-cap64-chunk=cap": (33, 64, 64, False, 12, {"chunk-of-capacity-into-non-empty", "empty-streams-between"}),
    "S33-cap256-chunk96": (33, 256, 96, False, 14, {"empty-streams-between"}),
    "S127-cap64-chunk=cap": (127, 64, 64, False, 10, {"chunk-of-capacity-into-non-empty", "empty-streams-between"}),
    "S127-cap256-chunk96": (127, 256, 96, False, 14, {"empty-streams-between"}),
    "S127-cap2^17-chunk512": (127, 1 << 17, 512, False, 6, {"empty-streams-between"}),
}


@pytest.mark.parametrize("name", list(RINGS))
def test_stream_push_and_ring_sort_follow_the_model(name):
    """the rings at 2^17 slots are not filled: the wrap and overflow paths are reached at 64 and 256 slots"""
    S, cap, mc, single, steps, extra = RINGS[name]
    assert S * cap < 1 << 24
    m = RingModel(S, cap, mc, single=single, sample=1 if single else 0)
    dev = DeviceRings(m, _geom(240, 180, 2 if single else S))
    big = cap > 4096
    seen = script(dev, steps, np.random.default_rng(S * 1000 + cap + mc), reset_at=steps - 4, fill=not big)
    need = (COMMON | extra) - ({"window-wraps", "overflow", "overflow-stays-set"} if big else set())
    assert need <= seen, sorted(need - seen)


def _ev(ts, x0=10):
    return [[x0 + (i % 7), 20 + (i % 5), int(t), 1] for i, t in enumerate(ts)]


def test_ring_flag_is_set_by_an_inversion_across_the_wrap_point():
    m = RingModel(1, 64, 64, single=True)
    dev = DeviceRings(m, _geom(240, 180, 1))
    dev.push(m.stage([[60, 0, 0, 0]], _ev(range(60))))
    ref = dev.check_sort("fill")
    assert not ref["flag"]
    dev.push(m.stage([[10, 50, 0, 0]], _ev([100, 101, 102, 103, 90, 91, 92, 93, 94, 95])))
    dev.check_rings("wrap")
    assert m.ctl[0] == 50 and m.pos[63, 2] == 103 and m.pos[0, 2] == 90       # the drop sits between slot 63 and slot 0
    ref = dev.check_sort("wrap")
    assert ref["flag"] and int(dev.sort.flags[0]) == 1


@pytest.mark.parametrize("S", [1, 3])
def test_ring_flag_ignores_an_evicted_slot_before_the_first_live_event(S):
    """a full ring, block 0 reset, then events with smaller t: the slot before the new head holds a larger, evicted t"""
    m = RingModel(S, 64, 64, single=S == 1)
    dev = DeviceRings(m, _geom(240, 180, S))
    dev.push(m.stage([[64, 0, 64 * s, 0] for s in range(S)], _ev(range(1000, 1000 + 64 * S))))
    dev.check_sort("full")
    dev.reset(0)
    dev.push(m.stage([[5, 0, 0, 0]] + [[0, 0, 0, 0]] * (S - 1), _ev(range(5))))
    dev.check_rings("after reset")
    assert m.ctl[0] == 0 and m.pos[63, 2] > m.pos[0, 2] and m.batch[63] == m.batch[0]
    ref = dev.check_sort("after reset")
    assert not ref["flag"] and int(dev.sort.flags[0]) == 0


def test_ring_flag_ignores_a_drop_across_two_streams():
    m = RingModel(2, 64, 32)
    dev = DeviceRings(m, _geom(240, 180, 2))
    dev.push(m.stage([[20, 0, 0, 0], [20, 0, 20, 0]], _ev(range(5000, 5020)) + _ev(range(20))))
    dev.check_rings("two streams")
    b, p, _ = m.windows()
    assert p[19, 2] > p[20, 2] and b[19] != b[20]
    ref = dev.check_sort("two streams")
    assert not ref["flag"] and int(dev.sort.flags[0]) == 0


# ------------------------------------------------------------------------------------------------------------------------
# input conversion
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H", [(640, 480), (1280, 720)])
def test_prepare_events_and_denormalize_pos_at_the_truncation_edges(W, H):
    L, lib = _lib()
    T = 1_000_000
    pos = edge_rows(W, H, T)
    N = len(pos)
    rng = np.random.default_rng(W)
    batch = rng.integers(-(1 << 40), 1 << 40, N)
    batch[:4] = [(1 << 32) + 5, -1, 1 << 31, -(1 << 31) - 1]
    d_pos = torch.from_numpy(pos).cuda()
    for ldx in (1, 3):
        x = rng.standard_normal((N, ldx)).astype(np.float32)
        pos_i, batch_i, feat = ref_prepare(pos, batch, x, ldx, W, H, T)
        o_pos = torch.full((N, 3), SENT, dtype=torch.int32, device="cuda")
        o_b = torch.full((N,), SENT, dtype=torch.int32, device="cuda")
        o_f = torch.full((N,), SENT, dtype=torch.int32, device="cuda")
        d_b, d_x = torch.from_numpy(batch).cuda(), torch.from_numpy(x).cuda()
        L.check(lib.dagr_prepare_events(P(d_pos), P(d_b), P(d_x), ldx, N, W, H, T, P(o_pos), P(o_b), P(o_f), st()), "prepare")
        torch.cuda.synchronize()
        assert torch.equal(o_pos.cpu(), torch.from_numpy(pos_i)), (W, H, ldx)
        assert torch.equal(o_b.cpu(), torch.from_numpy(batch_i)), (W, H, ldx)
        assert torch.equal(o_f.cpu(), torch.from_numpy(feat.copy()).view(torch.int32)), (W, H, ldx)
    o_pos = torch.full((N, 3), SENT, dtype=torch.int32, device="cuda")
    L.check(lib.dagr_denormalize_pos(P(d_pos), N, W, H, T, P(o_pos), st()), "denormalize")
    torch.cuda.synchronize()
    assert torch.equal(o_pos.cpu(), torch.from_numpy(pos_i))
