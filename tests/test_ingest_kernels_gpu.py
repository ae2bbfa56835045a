"""The batch event-ingest kernels of csrc/ingest.cu on their own, through the C-ABI, outputs pre-filled with sentinels:
  * dagr_downsample_events bit for bit against oracle/ref_ingest (pinned to the reference's numba down-sampler by
    downsample_golden.npz): N on either side of the 2048-element scan tile, grids on either side of 2048 cells and far
    larger than N, one cell holding every event, maps seeded at +-1, one ulp either side and +-(1 - k/d) at the inexact
    denominators 3 and 9 and at 8, and events past fx * out_w / fy * out_h against the kernel's clamp;
  * dagr_compact_events against events[mask != 0] with (x / fx, y / fy);
  * dagr_ingest_events bit for bit against the reference's own preprocessing chain (ingest_window_golden.npz, the
    unsorted and all-negative windows included) and on the exhaustive denormalisation sweep at absolute bases 0 and 7e9;
  * downsample + compact against dagr_stream_ingest on the same chunks, which share the accumulator step."""
import numpy as np
import pytest
import torch

from tests.test_ingest_kernels_cpu import WINDOW_GOLD, NCASES, sweep_events, sweep_expected, window_case

pytestmark = pytest.mark.gpu

TILE = 2048                                             # SCAN_TILE of csrc/graph.cu


def _lib():
    from dagr_b200 import _lib as L
    return L, L.load()


def _dev(a):
    """a host array as a device tensor; the caller keeps it alive until the call that reads it has run."""
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint16:
        a = a.view(np.int16)                            # the kernels read the u16 bit pattern
    return torch.from_numpy(a).cuda()


def map_seeds(d):
    """float32 accumulator values at the pass decision of denominator d: +-1, +-(1 - k/d) for k = 1..3 and +-(1 - 2^-24),
    each with its neighbours one ulp either side (tests/golden/make_downsample_golden.py seeds the golden maps alike)."""
    base = [np.float32(1)] + [np.float32(1 - k / d) for k in range(1, 4) if k < d] + [np.float32(1 - 2.0 ** -24)]
    v = np.array([w for b in base for w in (b, np.nextafter(b, np.float32(0)), np.nextafter(b, np.float32(2)))], np.float32)
    return np.unique(np.concatenate([v, -v]))


def seeded_map(rng, ow, oh, d, frac=1 / 3):
    s = map_seeds(d)
    m = np.zeros(oh * ow, np.float32)
    cells = rng.permutation(oh * ow)[:max(len(s), int(oh * ow * frac))]
    m[cells] = s[np.arange(len(cells)) % len(s)]
    return m.reshape(oh, ow), cells


def events(rng, n, fx, fy, ow, oh, cells=None, frac=0.8, xmax=None, ymax=None):
    """n events with x < fx * ow, y < fy * oh (or < xmax / ymax), p = +-1; a fraction `frac` on the output cells `cells`."""
    x = rng.integers(0, xmax or fx * ow, n)
    y = rng.integers(0, ymax or fy * oh, n)
    if cells is not None:
        on = rng.random(n) < frac
        c = cells[rng.integers(0, len(cells), on.sum())]
        x[on] = (c % ow) * fx + rng.integers(0, fx, on.sum())
        y[on] = (c // ow) * fy + rng.integers(0, fy, on.sum())
    return x.astype(np.uint16), y.astype(np.uint16), (2 * rng.integers(0, 2, n) - 1).astype(np.int8)


def downsample(x, y, p, fx, fy, ow, oh, cmap):
    """dagr_downsample_events; cmap float32[oh, ow] on the device, updated in place.  Returns the mask (host) after
    checking that every mask byte was written and that `count` is zero again."""
    L, lib = _lib()
    N, cells = len(x), ow * oh
    dev = "cuda"
    work = [torch.full((max(N, 1),), -7, dtype=torch.int32, device=dev) for _ in range(3)]
    count = torch.zeros(cells, dtype=torch.int32, device=dev)
    start = torch.full((cells + 1,), -7, dtype=torch.int32, device=dev)
    bs = torch.full((int(lib.dagr_scan_blocks(max(N, cells))) + 2,), -7, dtype=torch.int32, device=dev)
    mask = torch.full((N + 16,), 0xAA, dtype=torch.uint8, device=dev)
    dx, dy, dp = _dev(x), _dev(y), _dev(p)                      # held until the call has run
    L.check(lib.dagr_downsample_events(L.ptr(dx), L.ptr(dy), L.ptr(dp), N, fx, fy, ow, oh, L.ptr(cmap),
                                       *(L.ptr(w) for w in work), L.ptr(count), L.ptr(start), L.ptr(bs), L.ptr(mask),
                                       L.stream_ptr()), "downsample_events")
    m = mask.cpu().numpy()
    assert set(np.unique(m[:N])) <= {0, 1}, "a mask byte was not written"
    assert (m[N:] == 0xAA).all(), "written past N"
    assert not count.any(), "count is not zero on exit"
    return m[:N].astype(bool)


def oracle_downsample(x, y, p, fx, fy, ow, oh, m0):
    """oracle/ref_ingest's walk after the kernel's clamp of the output cell to (min(x / fx, ow - 1), min(y / fy, oh - 1)),
    the one place the test restates it (the reference would index out of bounds)."""
    from oracle import ref_ingest as R
    xl = np.minimum(x.astype(np.int64) // fx, ow - 1)
    yl = np.minimum(y.astype(np.int64) // fy, oh - 1)
    cm = m0.copy()
    mask = R.filter_events_resize(xl * fx, yl * fy, p, cm, fx, fy)
    return mask, cm


def check_downsample(x, y, p, fx, fy, ow, oh, m0):
    cmap = torch.from_numpy(m0.copy()).cuda()
    got = downsample(x, y, p, fx, fy, ow, oh, cmap)
    want, wm = oracle_downsample(x, y, p, fx, fy, ow, oh, m0)
    gm = cmap.cpu().numpy()
    assert np.array_equal(got, want)
    assert np.array_equal(gm.view(np.uint32), wm.view(np.uint32))
    hit = np.zeros(oh * ow, bool)
    hit[np.minimum(y.astype(np.int64) // fy, oh - 1) * ow + np.minimum(x.astype(np.int64) // fx, ow - 1)] = True
    assert np.array_equal(gm.reshape(-1)[~hit].view(np.uint32), m0.reshape(-1)[~hit].view(np.uint32)), "a cell without events changed"
    return got


@pytest.mark.parametrize("n", [1, TILE - 1, TILE, TILE + 1, 3 * TILE + 1])
def test_downsample_n_at_the_scan_tiles(n):
    rng = np.random.default_rng(n)
    ow, oh = 320, 240                                   # 76800 cells >> n
    for fx, fy in ((2, 2), (3, 1), (3, 3)):
        m0, cells = seeded_map(rng, ow, oh, fx * fy)
        x, y, p = events(rng, n, fx, fy, ow, oh, cells)
        check_downsample(x, y, p, fx, fy, ow, oh, m0)


@pytest.mark.parametrize("ow,oh", [(89, 23), (64, 32), (683, 3), (1, 1)])       # 2047, 2048, 2049 cells, and one cell
def test_downsample_cells_at_the_scan_tiles(ow, oh):
    rng = np.random.default_rng(ow * oh)
    for fx, fy in ((3, 1), (4, 2), (3, 3)):
        m0, cells = seeded_map(rng, ow, oh, fx * fy)
        x, y, p = events(rng, 5000, fx, fy, ow, oh, cells)
        check_downsample(x, y, p, fx, fy, ow, oh, m0)


def test_downsample_all_events_in_one_cell():
    """6145 events (more than 3 scan tiles) in one cell of 9 x 7: the one thread walks them in arrival order."""
    rng = np.random.default_rng(1)
    for fx, fy, d in ((3, 3, 9), (4, 2, 8), (3, 1, 3)):
        n = 3 * TILE + 1
        x = (4 * fx + rng.integers(0, fx, n)).astype(np.uint16)
        y = (2 * fy + rng.integers(0, fy, n)).astype(np.uint16)
        p = np.where(rng.random(n) < 0.6, 1, -1).astype(np.int8)
        seeds = map_seeds(d)
        for seed in (0.0, seeds[0], seeds[len(seeds) // 2], seeds[-1]):
            m0 = np.zeros((7, 9), np.float32)
            m0[2, 4] = seed
            mask = check_downsample(x, y, p, fx, fy, 9, 7, m0)
            assert 0 < mask.sum() < n


@pytest.mark.parametrize("fx,fy", [(3, 1), (4, 2), (3, 3), (1, 1), (2, 1)])
def test_downsample_seeded_maps_near_one(fx, fy):
    """every seed on its own cell, hit by one +1 and one -1 event in turn, then by random events over several chunks
    with the map carried over."""
    rng = np.random.default_rng(10 * fx + fy)
    d = fx * fy
    seeds = map_seeds(d)
    ow, oh = len(seeds), 2
    m0 = np.zeros((oh, ow), np.float32)
    m0[0] = seeds
    m0[1] = seeds
    x = np.concatenate([np.arange(ow) * fx, np.arange(ow) * fx + fx - 1]).astype(np.uint16)
    y = np.concatenate([np.zeros(ow), np.full(ow, 2 * fy - 1)]).astype(np.uint16)
    p = np.concatenate([np.ones(ow), -np.ones(ow)]).astype(np.int8)
    check_downsample(x, y, p, fx, fy, ow, oh, m0)
    cm = m0.copy()
    for _ in range(3):
        x, y, p = events(rng, 4000, fx, fy, ow, oh)
        cmap = torch.from_numpy(cm).cuda()
        got = downsample(x, y, p, fx, fy, ow, oh, cmap)
        want, cm = oracle_downsample(x, y, p, fx, fy, ow, oh, cm)
        assert np.array_equal(got, want) and np.array_equal(cmap.cpu().numpy().view(np.uint32), cm.view(np.uint32))


def test_downsample_clamps_events_past_the_grid():
    """x >= fx * out_w and y >= fy * out_h (up to 65535) land in the last column / row."""
    rng = np.random.default_rng(4)
    for fx, fy, ow, oh in ((3, 3, 40, 30), (4, 2, 32, 24), (3, 1, 7, 5)):
        m0, cells = seeded_map(rng, ow, oh, fx * fy)
        x, y, p = events(rng, 6000, fx, fy, ow, oh, cells, frac=0.3, xmax=65536, ymax=65536)
        x[:4], y[:4] = [65535, fx * ow, fx * ow - 1, 0], [65535, fy * oh, 0, fy * oh - 1]
        assert (x >= fx * ow).sum() > 1000 and (y >= fy * oh).sum() > 1000
        check_downsample(x, y, p, fx, fy, ow, oh, m0)


# ---------------------------------------------------------------------------------------------------------------------
def compact(mask, x, y, t, p, fx, fy):
    L, lib = _lib()
    N = len(mask)
    dev = "cuda"
    flag = torch.full((max(N, 1),), -7, dtype=torch.int32, device=dev)
    pos = torch.full((N + 1,), -7, dtype=torch.int32, device=dev)
    bs = torch.full((int(lib.dagr_scan_blocks(N)) + 2,), -7, dtype=torch.int32, device=dev)
    xo = torch.full((N + 8,), 0x5A5A, dtype=torch.int16, device=dev)
    yo = torch.full((N + 8,), 0x5A5A, dtype=torch.int16, device=dev)
    to = torch.full((N + 8,), -(1 << 40), dtype=torch.int64, device=dev)
    po = torch.full((N + 8,), 99, dtype=torch.int8, device=dev)
    n_out = torch.full((1,), -7, dtype=torch.int32, device=dev)
    dm, dx, dy, dt, dp = (_dev(a) for a in (mask, x, y, t, p))
    L.check(lib.dagr_compact_events(L.ptr(dm), N, L.ptr(dx), L.ptr(dy), L.ptr(dt), L.ptr(dp), fx, fy,
                                    L.ptr(flag), L.ptr(pos), L.ptr(bs), L.ptr(xo), L.ptr(yo), L.ptr(to), L.ptr(po), L.ptr(n_out),
                                    L.stream_ptr()), "compact_events")
    M = int(n_out.item())
    keep = mask != 0
    assert M == int(keep.sum())
    for got, fill in ((xo, 0x5A5A), (yo, 0x5A5A), (to, -(1 << 40)), (po, 99)):
        assert (got[M:] == fill).all(), "written past n_out"
    assert np.array_equal(xo[:M].cpu().numpy().view(np.uint16), (x[keep] // fx).astype(np.uint16))
    assert np.array_equal(yo[:M].cpu().numpy().view(np.uint16), (y[keep] // fy).astype(np.uint16))
    assert np.array_equal(to[:M].cpu().numpy(), t[keep]) and np.array_equal(po[:M].cpu().numpy(), p[keep])
    return M


def test_compact_masks():
    rng = np.random.default_rng(2)
    N = 5 * TILE + 37
    x = rng.integers(0, 65536, N).astype(np.uint16)
    y = rng.integers(0, 65536, N).astype(np.uint16)
    x[:3] = 65535
    t = rng.integers(-(1 << 40), 1 << 40, N).astype(np.int64)
    p = rng.integers(-128, 128, N).astype(np.int8)
    runs = np.zeros(N, np.uint8)                                   # runs of random length, some across the tiles
    i, v = 0, 1
    while i < N:
        ln = int(rng.integers(1, 3 * TILE))
        runs[i:i + ln] = v
        i, v = i + ln, 1 - v
    masks = {"zeros": np.zeros(N, np.uint8), "ones": np.ones(N, np.uint8), "alternate": (np.arange(N) & 1).astype(np.uint8),
             "runs": runs, "values": rng.choice(np.array([0, 1, 2, 255], np.uint8), N)}
    for fx, fy in ((1, 1), (2, 2), (3, 1), (3, 3), (4, 2)):
        for name, m in masks.items():
            M = compact(m, x, y, t, p, fx, fy)
            assert M == {"zeros": 0, "ones": N}.get(name, M), name
    assert compact(np.ones(1, np.uint8), np.array([65535], np.uint16), np.array([7], np.uint16), t[:1], p[:1], 3, 2) == 1
    for n in (1, TILE - 1, TILE, TILE + 1):
        compact(masks["values"][:n], x[:n], y[:n], t[:n], p[:n], 3, 3)


def test_compact_and_downsample_with_no_events():
    L, lib = _lib()
    n_out = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    pos, bs = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda")
    L.check(lib.dagr_compact_events(None, 0, None, None, None, None, 2, 2, None, L.ptr(pos), L.ptr(bs), None, None, None, None,
                                    L.ptr(n_out), L.stream_ptr()), "compact_events")
    assert int(n_out.item()) == 0
    cm = torch.full((3, 4), 0.5, dtype=torch.float32, device="cuda")
    assert not downsample(np.zeros(0, np.uint16), np.zeros(0, np.uint16), np.zeros(0, np.int8), 2, 2, 4, 3, cm).size
    assert bool((cm == 0.5).all())


# ---------------------------------------------------------------------------------------------------------------------
def ingest(ev, W, H, T, t_cut, p_is_01=True, sample=3):
    """dagr_ingest_events on host arrays -> (pos i32[M, 3], feat f32[M]), after checking batch and the sentinels past M."""
    L, lib = _lib()
    N = len(ev["t"])
    dev = "cuda"
    flag = torch.full((max(N, 1),), -7, dtype=torch.int32, device=dev)
    pos = torch.full((N + 1,), -7, dtype=torch.int32, device=dev)
    bs = torch.full((int(lib.dagr_scan_blocks(N)) + 2,), -7, dtype=torch.int32, device=dev)
    tlast = torch.full((1,), 12345, dtype=torch.int64, device=dev)
    batch = torch.full((N + 4,), -7, dtype=torch.int32, device=dev)
    pos_o = torch.full((N + 4, 3), -7, dtype=torch.int32, device=dev)
    feat = torch.full((N + 4,), -7.0, dtype=torch.float32, device=dev)
    n_out = torch.full((1,), -7, dtype=torch.int32, device=dev)
    p = ev["p"].astype(np.int8) if p_is_01 else (2 * ev["p"].astype(np.int8) - 1)
    dx, dy, dt, dp = _dev(ev["x"]), _dev(ev["y"]), _dev(ev["t"]), _dev(p)
    L.check(lib.dagr_ingest_events(L.ptr(dx), L.ptr(dy), L.ptr(dt), L.ptr(dp), N,
                                   1 if p_is_01 else 0, W, H, T, int(t_cut), sample, L.ptr(flag), L.ptr(pos), L.ptr(bs), L.ptr(tlast),
                                   L.ptr(batch), L.ptr(pos_o), L.ptr(feat), L.ptr(n_out), L.stream_ptr()), "ingest_events")
    M = int(n_out.item())
    assert (batch[:M] == sample).all() and (batch[M:] == -7).all() and (pos_o[M:] == -7).all() and (feat[M:] == -7.0).all()
    return pos_o[:M].cpu().numpy(), feat[:M].cpu().numpy()


@pytest.mark.parametrize("p_is_01", [1, 0])
@pytest.mark.parametrize("case", range(NCASES))
def test_ingest_equals_reference_golden(case, p_is_01):
    """c9 (unsorted) and c10 (all negative) take t[-1] from the last kept event in array order, as the reference does."""
    g = np.load(WINDOW_GOLD)
    ev, W, H, T, cut, want_pos, want_feat = window_case(g, case)
    pos, feat = ingest(ev, W, H, T, cut, p_is_01=bool(p_is_01))
    assert pos.shape == want_pos.shape
    bad = np.flatnonzero((pos != want_pos).any(1))
    assert not len(bad), f"{len(bad)} of {len(pos)} rows differ, first row {bad[0]}: {pos[bad[0]]} != {want_pos[bad[0]]}"
    assert np.array_equal(feat, want_feat)


def test_ingest_exhaustive_denormalisation_sweep():
    """every t in [0, T], x < W and y < H of the fixture's sweep, at absolute bases 0 and 7e9, p_is_01 = 1 and 0: the
    reference's values (the stored truncations included) and the oracle's."""
    from oracle import ref_ingest as R
    g = np.load(WINDOW_GOLD)
    for k, (W, H, T) in enumerate(tuple(int(v) for v in d) for d in g["sweep_dims"]):
        want = sweep_expected(g, W, H, T)
        for base in (0, 7_000_000_000):
            ev = sweep_events(W, H, T, base)
            p01 = (k + base // 7_000_000_000) % 2 == 0
            pos, feat = ingest(ev, W, H, T, 1 << 62, p_is_01=p01)
            assert np.array_equal(pos, want), (W, H, T, base)
            assert np.array_equal(feat, (2 * ev["p"].astype(np.float32) - 1)), (W, H, T, base)
            if base:
                den, pol = R.preprocess_window(ev, W, H, T)
                assert np.array_equal(pos, den) and np.array_equal(feat, pol)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fx,fy", [(3, 1), (4, 2), (3, 3)])
def test_downsample_compact_equals_stream_ingest(fx, fy):
    """the same chunks, the map carried over n = 1, 1023, 1024, 1025 and 16384 events from a seeded map: downsample +
    compact and dagr_stream_ingest give the same rows and the same map bits."""
    from dagr_b200 import _lib as L
    from dagr_b200.streaming import pack_raw_stage
    lib = L.load()
    rng = np.random.default_rng(fx * 10 + fy)
    ow, oh, MR = 64, 48, 16384
    m0, cells = seeded_map(rng, ow, oh, fx * fy)
    cm_a = torch.from_numpy(m0.copy()).cuda()
    cm_b = torch.from_numpy(m0.copy()).cuda().view(1, oh, ow)
    raw = np.zeros(4 + 2 * MR, np.int32)
    for n in (1, 1023, 1024, 1025, 16384):
        x, y, p = events(rng, n, fx, fy, ow, oh, cells)
        t = np.sort(rng.integers(0, 1 << 30, n)).astype(np.int64)
        mask = downsample(x, y, p, fx, fy, ow, oh, cm_a)
        keep = mask.astype(np.uint8)
        compact(keep, x, y, t, p, fx, fy)                          # checks the rows against events[mask] itself
        pack_raw_stage(raw, [(x, y, t, p)], [0], MR)
        stage = torch.full((4 + 4 * MR,), -9, dtype=torch.int32, device="cuda")
        draw = torch.from_numpy(raw).cuda()
        L.check(lib.dagr_stream_ingest(L.ptr(draw), 1, MR, fx, fy, ow, oh, oh, L.ptr(cm_b), L.ptr(stage), MR,
                                       L.stream_ptr()), "stream_ingest")
        s = stage.cpu().numpy()
        rows = s[4:4 + 4 * int(s[0])].reshape(-1, 4)
        assert int(s[0]) == int(mask.sum()), n
        want = np.stack([x[mask] // fx, y[mask] // fy, t[mask], p[mask]], 1).astype(np.int32)
        assert np.array_equal(rows, want), n
        assert np.array_equal(cm_a.cpu().numpy().view(np.uint32), cm_b[0].cpu().numpy().view(np.uint32)), n
