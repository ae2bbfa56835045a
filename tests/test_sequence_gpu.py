"""SequenceDetector: many time windows of one recording as the samples of batched forwards.  The gather kernel must equal
numpy bit for bit; every window's detections must equal, bit for bit, a streaming detector pushed with chunks cut at the
query times (events-only, raw sensor, image fusion) and model(data) at B = 1 over the window's events (with the window's
frame); the bits must not depend on the blocking or on the engine's overlap mode; each frame runs through the trunk once
per call; and the block loop makes no host synchronisation."""
import numpy as np
import pytest
import torch

from tests.helpers import make_model

pytestmark = pytest.mark.gpu

W, H = 320, 215
SW, SH = 640, 480
WINDOW = 20_000


def _same(a, b):
    return (len(a["boxes"]) == len(b["boxes"]) and torch.equal(a["boxes"].cpu(), b["boxes"].cpu())
            and torch.equal(a["scores"].cpu(), b["scores"].cpu()) and torch.equal(a["labels"].cpu(), b["labels"].cpu()))


def _dense(model, x, y, t, p, frame=None):
    """model(data) at B = 1 over one window's events (pos_denorm = the events), with the frame normalised as format_data."""
    from dagr_b200.data import EventBatch
    n = len(t)
    pos = torch.from_numpy(np.stack([x, y, t], 1).astype(np.int32).reshape(n, 3)).cuda()
    feat = torch.from_numpy(np.asarray(p, np.float32)).cuda()
    kw = {} if frame is None else dict(image=frame.cuda().float().unsqueeze(0) / 255.0)
    d = EventBatch(x=feat.view(-1, 1), pos=torch.zeros(n, 3, device="cuda"), batch=torch.zeros(n, dtype=torch.long, device="cuda"),
                   width=torch.tensor([W]), height=torch.tensor([H]), time_window=torch.tensor([1_000_000]), pos_denorm=pos,
                   num_graphs=1, dims=(W, H, 1_000_000), **kw)
    return model(d)[0][0]


def _recording(rate, seconds, seed, kind, gap=None, t0=0):
    """host arrays (x, y int16, t int32, p int8 +-1) of a synthetic recording; `gap` = (a_us, b_us) without events."""
    from dagr_b200.streaming import synth_stream
    x, y, t, p = synth_stream(rate, seconds, W, H, seed=seed, kind=kind)
    keep = np.ones(len(t), bool) if gap is None else ~((t >= gap[0]) & (t < gap[1]))
    return dict(x=x[keep], y=y[keep], t=(t[keep].astype(np.int64) + t0).astype(np.int32), p=p[keep])


def _stream_reference(make_det, ev, t_end, before_push=None):
    """detections of a streaming detector pushed with chunks cut at the sorted distinct query times: chunk k = the events of
    [t_{k-1}, t_k) with t_end = t_k.  A push evicts before it appends, so a chunk that also holds events older than
    t_k - WINDOW is pushed in two, the older part first with t_end = t_k - WINDOW; then every step's live window is exactly
    [t_k - WINDOW, t_k).  Returns one result per query, in the query order."""
    det = make_det()
    t = ev["t"]
    out, prev = {}, None
    for te in np.unique(t_end):
        a = 0 if prev is None else np.searchsorted(t, prev)
        m, b = np.searchsorted(t, [te - WINDOW, te])
        if before_push is not None:
            before_push(det, te)
        if m > a:
            det.push(ev["x"][a:m], ev["y"][a:m], t[a:m], ev["p"][a:m], int(te - WINDOW))
            a = m
        out[int(te)] = det.push(ev["x"][a:b], ev["y"][a:b], t[a:b], ev["p"][a:b], int(te))[0]
        prev = te
    return [out[int(te)] for te in t_end]


@pytest.fixture(scope="module")
def model():
    return make_model("s", H, W, batch_size=1)[0].cuda()


@pytest.fixture(scope="module")
def hybrid():
    return make_model("s", H, W, batch_size=1, use_image=True, img_net="resnet18")[0].cuda()


# ---- 1. the kernels ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p01,t_base", [(0, 0), (1, 4_000_000_123)])
def test_bounds_and_gather_equal_numpy(p01, t_base):
    from dagr_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(3)
    N = 50_000
    t = np.sort(rng.integers(0, 30_000, N)).astype(np.int64) + t_base        # ~1.7 events per us: many duplicates
    x = rng.integers(0, 65536, N).astype(np.uint16)
    y = rng.integers(0, 32768, N).astype(np.uint16)
    p = (rng.integers(0, 2, N) if p01 else rng.choice([-1, 1], N)).astype(np.int8)
    a = lambda v: int(v) + t_base
    tb = np.array([a(0), a(100), a(100), a(-50), a(29_990), a(5_000), a(7), a(40_000), a(1_000), int(t[500]), int(t[-1])], np.int64)
    te = np.array([a(0), a(2_000), a(2_000), a(10), a(31_000), a(25_000), a(8), a(50_000), a(1_000), int(t[900]), int(t[-1]) + 1], np.int64)
    G = len(tb)
    assert (t == tb[-2]).any() and (t == te[-2]).any()                      # events exactly at a t_begin and at a t_end
    d = lambda v: torch.from_numpy(v).cuda()
    dt, dx, dy, dp = d(t), d(x.view(np.int16)), d(y.view(np.int16)), d(p)
    begin, end = torch.empty(G, dtype=torch.int32, device="cuda"), torch.empty(G, dtype=torch.int32, device="cuda")
    dtb, dte = d(tb), d(te)
    _lib.check(lib.dagr_window_bounds(_lib.ptr(dt), N, _lib.ptr(dtb), _lib.ptr(dte), G, _lib.ptr(begin), _lib.ptr(end), _lib.stream_ptr()))
    wb, we = np.searchsorted(t, tb, "left"), np.searchsorted(t, te, "left")
    assert np.array_equal(begin.cpu().numpy(), wb) and np.array_equal(end.cpu().numpy(), we)
    sizes = we - wb
    total = int(sizes.sum())
    batch = torch.full((total + 7,), -7, dtype=torch.int32, device="cuda")
    pos = torch.full((total + 7, 3), -7, dtype=torch.int32, device="cuda")
    feat = torch.full((total + 7,), -7.0, dtype=torch.float32, device="cuda")
    offs = torch.empty(G + 1, dtype=torch.int64, device="cuda")
    _lib.check(lib.dagr_window_gather(_lib.ptr(dx), _lib.ptr(dy), _lib.ptr(dt), _lib.ptr(dp), N, _lib.ptr(begin), _lib.ptr(end), G, t_base,
                                      p01, total, _lib.ptr(batch), _lib.ptr(pos), _lib.ptr(feat), _lib.ptr(offs), _lib.stream_ptr()))
    idx = np.concatenate([np.arange(b, e) for b, e in zip(wb, we)])
    assert np.array_equal(offs.cpu().numpy(), np.concatenate([[0], np.cumsum(sizes)]))
    assert np.array_equal(batch.cpu().numpy()[:total], np.repeat(np.arange(G), sizes))
    want_pos = np.stack([x[idx].astype(np.int32), y[idx].astype(np.int32), (t[idx] - t_base).astype(np.int32)], 1)
    assert np.array_equal(pos.cpu().numpy()[:total], want_pos)
    want_feat = (2 * p[idx].astype(np.int32) - 1 if p01 else p[idx]).astype(np.float32)
    assert np.array_equal(feat.cpu().numpy()[:total], want_feat)
    assert (batch.cpu().numpy()[total:] == -7).all() and (pos.cpu().numpy()[total:] == -7).all()   # nothing past the total
    # the rows bound: a smaller total writes a prefix only
    batch.fill_(-7)
    _lib.check(lib.dagr_window_gather(_lib.ptr(dx), _lib.ptr(dy), _lib.ptr(dt), _lib.ptr(dp), N, _lib.ptr(begin), _lib.ptr(end), G, t_base,
                                      p01, 1000, _lib.ptr(batch), _lib.ptr(pos), _lib.ptr(feat), _lib.ptr(offs), _lib.stream_ptr()))
    bh = batch.cpu().numpy()
    assert np.array_equal(bh[:1000], np.repeat(np.arange(G), sizes)[:1000]) and (bh[1000:] == -7).all()


# ---- 2.-4. events only ------------------------------------------------------------------------------------------------
def _cases():
    rng = np.random.default_rng(11)
    irregular = np.sort(rng.integers(2_000, 150_000, 40))
    irregular = np.concatenate([irregular, irregular[::7]])                  # duplicates
    rng.shuffle(irregular)                                                   # unsorted query order
    return {
        "uniform_grid": (_recording(300_000, 0.15, 5, "uniform"), np.arange(10_000, 150_001, 1_000)),
        "clustered_grid": (_recording(400_000, 0.15, 6, "clustered"), np.arange(10_000, 150_001, 1_000)),
        "irregular_duplicates": (_recording(300_000, 0.15, 7, "clustered"), irregular),
        "gap": (_recording(300_000, 0.15, 8, "uniform", gap=(40_000, 100_000)), np.arange(30_000, 150_001, 2_500)),
    }


CASES = _cases()


@pytest.mark.parametrize("case", sorted(CASES))
def test_events_only_windows_equal_streaming_detector(model, case):
    from dagr_b200.sequence import SequenceDetector
    from dagr_b200.streaming import StreamingDetector
    ev, t_end = CASES[case]
    det = SequenceDetector(model, window_us=WINDOW, max_windows=32)
    got = det.detect(ev, t_end)
    want = _stream_reference(lambda: StreamingDetector(model, window_us=WINDOW, max_chunk=1 << 16, capacity=1 << 17), ev, t_end)
    assert len(got) == len(t_end)
    bad = [q for q in range(len(t_end)) if not _same(got[q], want[q])]
    assert not bad, (case, bad[:5])
    assert sum(len(g["boxes"]) for g in got) > 0
    assert got[0]["boxes"].is_cuda
    d, n = det.last
    assert d.shape[0] == n.shape[0] == len(t_end) and n.cpu().tolist() == [len(g["boxes"]) for g in got]
    if case == "gap":                                                          # windows inside the gap are empty: one answer
        inside = [q for q, te in enumerate(t_end) if te - WINDOW >= 40_000 and te <= 100_000]
        assert len(inside) > 1 and all(_same(got[q], got[inside[0]]) for q in inside)


def test_events_only_windows_equal_dense_forward(model):
    from dagr_b200.sequence import SequenceDetector
    ev, t_end = CASES["irregular_duplicates"]
    tb = t_end - np.array([WINDOW, 5_000, 33_000, 1] * (len(t_end) // 4 + 1))[:len(t_end)]    # anchored windows of any length
    got = SequenceDetector(model, window_us=WINDOW, max_windows=16).detect(ev, t_end, t_begin=tb)
    for q in range(0, len(t_end), 6):
        a, b = np.searchsorted(ev["t"], [tb[q], t_end[q]])
        want = _dense(model, ev["x"][a:b], ev["y"][a:b], ev["t"][a:b], ev["p"][a:b])
        assert _same(got[q], want), q


def test_blocking_and_overlap_do_not_change_the_bits(model):
    from dagr_b200.sequence import SequenceDetector
    ev, t_end = CASES["clustered_grid"]
    ref = SequenceDetector(model, window_us=WINDOW, max_windows=64).detect(ev, t_end)
    runs = {}
    for mw, me in ((1, 1 << 23), (7, 1 << 23), (64, 15_000)):                 # 15 k events: blocks of a few windows
        runs[(mw, me)] = SequenceDetector(model, window_us=WINDOW, max_windows=mw, max_events=me).detect(ev, t_end)
    twin = make_model("s", H, W, batch_size=1)[0].cuda()                       # the same weights, an engine of its own
    twin.engine.overlap = True
    runs["overlap"] = SequenceDetector(twin, window_us=WINDOW, max_windows=7).detect(ev, t_end)
    for k, got in runs.items():
        assert all(_same(a, b) for a, b in zip(got, ref)), k


def test_block_loop_makes_no_host_sync(model, monkeypatch):
    from dagr_b200.sequence import SequenceDetector
    ev, t_end = CASES["uniform_grid"]
    det = SequenceDetector(model, window_us=WINDOW, max_windows=8)
    ref = det.detect(ev, t_end)                                                # warm: packs, geometry, captured coarse stack
    inner = SequenceDetector._run_blocks
    calls = []

    def guarded(self, *a, **k):
        torch.cuda.set_sync_debug_mode("error")
        try:
            return inner(self, *a, **k)
        finally:
            torch.cuda.set_sync_debug_mode(0)
            calls.append(1)

    monkeypatch.setattr(SequenceDetector, "_run_blocks", guarded)
    got = det.detect(ev, t_end)
    assert calls == [1] and all(_same(a, b) for a, b in zip(got, ref))


# ---- 5. raw sensor ----------------------------------------------------------------------------------------------------
def test_raw_sensor_windows_equal_raw_streaming_detector(model):
    from dagr_b200.sequence import SequenceDetector
    from dagr_b200.streaming import synth_stream, StreamingDetector
    x, y, t, _ = synth_stream(1_500_000, 0.08, SW, SH, seed=5, kind="clustered")
    t0 = (1 << 31) + 123_456                                                  # raw timestamps above 2^31 us
    p = (np.random.default_rng(5).random(len(t)) < 0.85).astype(np.int8)
    ev = dict(x=x.astype(np.uint16), y=y.astype(np.uint16), t=t.astype(np.int64) + t0, p=p)
    t_end = t0 + np.concatenate([np.arange(2_000, 80_001, 2_000), [33_333, 33_333, 70_001]])
    det = SequenceDetector(model, window_us=WINDOW, max_windows=16, max_events=20_000, sensor=(SW, SH))   # 6 down-sampler slices
    got = det.detect(ev, t_end)
    want = _stream_reference(lambda: StreamingDetector(model, window_us=WINDOW, max_chunk=16384, capacity=1 << 15, sensor=(SW, SH)),
                             ev, t_end)
    bad = [q for q in range(len(t_end)) if not _same(got[q], want[q])]
    assert not bad, bad[:5]
    assert sum(len(g["boxes"]) for g in got) > 0


# ---- 6. image fusion --------------------------------------------------------------------------------------------------
def _frames(n, shape, seed=3):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n,) + shape, generator=g, dtype=torch.uint8)


def _fusion_reference(model, ev, t_end, frames, frame_t, **kw):
    from dagr_b200.streaming import FusionStreamingDetector
    state = dict(next=0)

    def before(det, te):                                                      # every frame with frame_t <= t_end, synced
        while state["next"] < len(frame_t) and frame_t[state["next"]] <= te:
            det.set_frame(frames[state["next"]])
            det.sync_frame()
            state["next"] += 1

    return _stream_reference(lambda: FusionStreamingDetector(model, window_us=WINDOW, max_chunk=1 << 16 if "sensor" not in kw else 16384,
                                                             capacity=1 << 17, **kw), ev, t_end, before)


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_fusion_windows_equal_fusion_streaming_detector(hybrid, precision, monkeypatch):
    from dagr_b200.model.image_branch import ImageBranch
    from dagr_b200.sequence import SequenceDetector
    hybrid.image_precision = precision
    try:
        ev = _recording(300_000, 0.12, 9, "clustered")
        frame_t = np.array([0, 20_000, 40_000, 60_000, 80_000, 100_000])
        frames = _frames(len(frame_t), (3, H, W))
        t_end = np.arange(4_000, 120_001, 4_000)
        det = SequenceDetector(hybrid, window_us=WINDOW, max_windows=8)
        runs = []
        real = ImageBranch.run
        monkeypatch.setattr(ImageBranch, "run", lambda self, *a, **k: (runs.append(1), real(self, *a, **k))[1])
        got = det.detect(ev, t_end, frames=frames, frame_t=frame_t)
        assert len(runs) == len(frame_t)                                       # 4 blocks, each frame through the trunk once
        monkeypatch.setattr(ImageBranch, "run", real)
        want = _fusion_reference(hybrid, ev, t_end, frames, frame_t)
        bad = [q for q in range(len(t_end)) if not _same(got[q], want[q])]
        assert not bad, bad[:5]
    finally:
        hybrid.image_precision = "tf32"


def test_fusion_raw_frames_equal_fusion_streaming_detector(hybrid):
    from dagr_b200.sequence import SequenceDetector
    from dagr_b200.streaming import synth_stream
    x, y, t, _ = synth_stream(1_500_000, 0.06, SW, SH, seed=12, kind="uniform")
    p = (np.random.default_rng(12).random(len(t)) < 0.85).astype(np.int8)
    t0 = 5_000_000_000
    ev = dict(x=x.astype(np.uint16), y=y.astype(np.uint16), t=t.astype(np.int64) + t0, p=p)
    frame_t = t0 + np.array([0, 25_000, 50_000])
    frames = _frames(len(frame_t), (SH, SW, 3), seed=4)
    t_end = t0 + np.arange(3_000, 60_001, 3_000)
    det = SequenceDetector(hybrid, window_us=WINDOW, max_windows=8, sensor=(SW, SH), raw_frames=True)
    got = det.detect(ev, t_end, frames=frames.numpy(), frame_t=frame_t)
    want = _fusion_reference(hybrid, ev, t_end, frames, frame_t, sensor=(SW, SH), raw_frames=True)
    bad = [q for q in range(len(t_end)) if not _same(got[q], want[q])]
    assert not bad, bad[:5]


def test_interframe_windows_equal_dense_forward_with_their_frame(hybrid):
    from dagr_b200.sequence import SequenceDetector, interframe_windows
    ev = _recording(300_000, 0.2, 10, "uniform")
    frame_t = np.array([10_000, 60_000, 110_000])
    frames = _frames(len(frame_t), (3, H, W), seed=6)
    tb, te, fi = interframe_windows(frame_t, steps=5, span_us=50_000)
    got = SequenceDetector(hybrid, max_windows=6).detect(ev, te, t_begin=tb, frames=frames.cuda(), frame_idx=fi)
    for q in range(len(te)):                                                   # the first window of each frame is empty
        a, b = np.searchsorted(ev["t"], [tb[q], te[q]])
        want = _dense(hybrid, ev["x"][a:b], ev["y"][a:b], ev["t"][a:b], ev["p"][a:b], frames[fi[q]])
        assert _same(got[q], want), q
