"""MultiStreamDetector: S event cameras as the S samples of one streaming step (one CUDA graph replay).  Each stream's
detections must equal, bit for bit, the synchronous forward over its live window and a single-stream StreamingDetector fed
the same chunks -- whatever the other streams do (different rates and time bases, empty chunks, a reset, an overflow)."""
import numpy as np
import pytest
import torch

from tests.helpers import make_model

pytestmark = pytest.mark.gpu

W, H = 320, 215
WINDOW, CHUNK, STEPS = 20_000, 2_000, 30
CHECKS = (0, 1, 2, 5, 11, 12, 13, 16, 20, 29)          # eager (0, 1) and replayed steps, before and after the window fills


def _stream(rate, seed, kind, t0=0, gap=None):
    """host arrays of one synthetic stream starting at t0 us; `gap` = (first, last + 1) step without events."""
    from dagr_b200.streaming import synth_stream
    x, y, t, p = synth_stream(rate, STEPS * CHUNK * 1e-6, W, H, seed=seed, kind=kind)
    keep = np.ones(len(t), bool) if gap is None else ~((t >= gap[0] * CHUNK) & (t < gap[1] * CHUNK))
    return x[keep], y[keep], (t[keep].astype(np.int64) + t0).astype(np.int32), p[keep], t0


def _chunk(ev, k):
    x, y, t, p, t0 = ev
    a, b = np.searchsorted(t, [t0 + k * CHUNK, t0 + (k + 1) * CHUNK])
    return x[a:b], y[a:b], t[a:b], p[a:b]


def _t_end(ev, k):
    return ev[4] + (k + 1) * CHUNK


def _same(a, b):
    return (len(a["boxes"]) == len(b["boxes"]) and torch.equal(a["boxes"], b["boxes"].cpu()) and torch.equal(a["scores"], b["scores"].cpu())
            and torch.equal(a["labels"], b["labels"].cpu()))


def _dense(model, pos, feat):
    """the synchronous forward over one live window (as test_streaming_window_equals_dense_forward_on_live_window)."""
    from dagr_b200.data import EventBatch
    n = len(feat)
    d = EventBatch(x=feat.view(-1, 1).clone(), pos=torch.zeros(n, 3, device="cuda"), batch=torch.zeros(n, dtype=torch.long, device="cuda"),
                   width=torch.tensor([W]), height=torch.tensor([H]), time_window=torch.tensor([1_000_000]),
                   pos_denorm=pos.clone(), num_graphs=1, dims=(W, H, 1_000_000))
    return model(d)[0][0]


def _heterogeneous():
    # 400 k / 150 k / 50 k ev/s; stream 1 lives 5 s later; stream 2 has no events for steps 14..18
    return [_stream(400_000, 5, "clustered"), _stream(150_000, 6, "uniform", t0=5_000_000),
            _stream(50_000, 7, "clustered", gap=(14, 19))]


def _chunks(evs, k):
    out = []
    for s, ev in enumerate(evs):
        c = _chunk(ev, k)
        out.append(None if len(c[2]) == 0 and k % 2 == 0 else c)           # both forms of "no events this step"
    return out


def test_multistream_live_windows_equal_dense_forward():
    from dagr_b200.streaming import MultiStreamDetector
    model, _ = make_model("s", H, W, batch_size=1)
    model.cuda()
    evs = _heterogeneous()
    S = len(evs)
    det = MultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    evicted_seen = [0] * S
    checked = 0
    for k in range(STEPS):
        out = det.push(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
        assert len(out) == S
        if k not in CHECKS:
            continue
        for s, ev in enumerate(evs):
            t, te = ev[2], _t_end(ev, k)
            live = (t >= te - WINDOW) & (t < te)
            gone = (t >= te - CHUNK - WINDOW) & (t < te - WINDOW) if k > 0 else np.zeros(len(t), bool)   # live one step ago
            st = det.window_state(s)
            assert st["live"] == int(live.sum()) and not st["overflow"], (k, s, st, int(live.sum()))
            assert st["appended"] == len(_chunk(ev, k)[2])
            assert st["evicted"] == int(gone.sum()), (k, s, st, int(gone.sum()))
            if k >= 11 and st["evicted"] > 0:
                evicted_seen[s] += 1
            pos, feat = det.live_window(s)
            assert np.array_equal(pos[:, 2].cpu().numpy(), t[live])
            assert np.array_equal(pos[:, 0].cpu().numpy(), ev[0][live].astype(np.int32))
            assert np.array_equal(feat.cpu().numpy(), ev[3][live].astype(np.float32))
            want = _dense(model, pos, feat)
            assert _same(out[s], want), (k, s, len(out[s]["boxes"]), len(want["boxes"]))
            checked += 1
    assert checked == S * len(CHECKS) and det.graph is not None
    assert min(evicted_seen) >= 3, evicted_seen


def test_multistream_equals_single_stream_detectors_every_step():
    from dagr_b200.streaming import MultiStreamDetector, StreamingDetector
    model, _ = make_model("s", H, W, batch_size=1)
    model.cuda()
    evs = _heterogeneous()
    S = len(evs)
    det = MultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    refs = [StreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15) for _ in range(S)]
    for k in range(STEPS):
        out = det.push(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
        for s, ev in enumerate(evs):
            want = refs[s].push(*_chunk(ev, k), _t_end(ev, k))[0]
            assert _same(out[s], want), (k, s, len(out[s]["boxes"]), len(want["boxes"]))
            assert det.window_state(s) == refs[s].window_state
    assert det.graph is not None and all(r.graph is not None for r in refs)


def test_multistream_reset_of_one_stream_leaves_the_others_alone():
    from dagr_b200.streaming import MultiStreamDetector, StreamingDetector
    model, _ = make_model("s", H, W, batch_size=1)
    model.cuda()
    evs = _heterogeneous()
    S, R = len(evs), 12
    fresh = _stream(200_000, 11, "uniform", t0=9_000_000)
    det = MultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    refs = [StreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15) for _ in range(S)]
    for k in range(STEPS):
        if k == R:                                        # stream 1 is handed to another camera
            det.reset(1)
            evs[1] = fresh
            refs[1] = StreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
        out = det.push(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
        for s, ev in enumerate(evs):
            want = refs[s].push(*_chunk(ev, k), _t_end(ev, k))[0]
            assert _same(out[s], want), (k, s, len(out[s]["boxes"]), len(want["boxes"]))
            assert det.window_state(s) == refs[s].window_state, (k, s)
    live = (fresh[2] >= _t_end(fresh, STEPS - 1) - WINDOW) & (fresh[2] < _t_end(fresh, STEPS - 1))
    assert det.window_state(1)["live"] == int(live.sum())


def test_multistream_overflow_of_one_stream_is_isolated():
    from dagr_b200.streaming import MultiStreamDetector, StreamingDetector
    model, _ = make_model("s", H, W, batch_size=1)
    model.cuda()
    cap = 1 << 12
    # stream 1 bursts at 400 k ev/s: ~8000 events per 20 ms window in a ring of 4096 slots
    evs = [_stream(100_000, 21, "uniform"), _stream(400_000, 22, "clustered", t0=1_000_000), _stream(50_000, 23, "uniform")]
    S = len(evs)
    det = MultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=2048, capacity=cap)
    refs = [StreamingDetector(model, window_us=WINDOW, max_chunk=2048, capacity=cap) for _ in range(S)]
    for k in range(STEPS):
        out = det.push([_chunk(ev, k) for ev in evs], [_t_end(ev, k) for ev in evs])
        for s, ev in enumerate(evs):
            want = refs[s].push(*_chunk(ev, k), _t_end(ev, k))[0]
            assert _same(out[s], want), (k, s)
    assert [det.window_state(s)["overflow"] for s in range(S)] == [False, True, False]
    assert det.window_state(1)["live"] == cap
    for s in (0, 2):                                      # the streams beside the burst still see their exact live window
        t, te = evs[s][2], _t_end(evs[s], STEPS - 1)
        live = (t >= te - WINDOW) & (t < te)
        pos, feat = det.live_window(s)
        assert np.array_equal(pos[:, 2].cpu().numpy(), t[live])
        assert _same(out[s], _dense(model, pos, feat))
