"""Raw sensor streaming: the detectors take a 640x480 camera's own events and run the reference's 2x down-sampler
(scripts/downsample_events.py), the crop to the model's height, the polarity 2p - 1 and the time rebase inside the step
(dagr_stream_ingest).  The kernel must equal the reference's own numba down-sampler bit for bit (golden vectors), and a
raw-mode detector must equal, bit for bit, a plain detector fed the chunks that oracle/ref_ingest builds on the host."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests.helpers import make_model
from tests.test_multistream_gpu import _same

pytestmark = pytest.mark.gpu

SW, SH = 640, 480                                     # the DSEC sensor
W, H = 320, 215                                       # the model: 2x down-sampled, cropped to 215 rows
WINDOW, CHUNK, STEPS = 20_000, 2_000, 30
GOLD_PATH = Path(__file__).resolve().parent / "golden" / "downsample_golden.npz"


def _raw_stream(rate, seed, kind="clustered", t0=0, seconds=STEPS * CHUNK * 1e-6, gap=None, positive=0.85):
    """host arrays of one synthetic raw camera stream: x, y uint16 at 640x480, t int64 us from t0, p in {0, 1}.  A fraction
    `positive` of the events is positive: with uniform random polarities the down-sampler keeps about 1 in 16 events at
    2x2, biased ones give the model a denser window."""
    from dagr_b200.streaming import synth_stream
    x, y, t, _ = synth_stream(rate, seconds, SW, SH, seed=seed, kind=kind)
    p = (np.random.default_rng(seed).random(len(t)) < positive).astype(np.int8)
    keep = np.ones(len(t), bool) if gap is None else ~((t >= gap[0] * CHUNK) & (t < gap[1] * CHUNK))
    return x[keep].astype(np.uint16), y[keep].astype(np.uint16), t[keep].astype(np.int64) + t0, p[keep], t0


def _cut(ev, a_us, b_us):
    x, y, t, p, t0 = ev
    a, b = np.searchsorted(t, [t0 + a_us, t0 + b_us])
    return x[a:b], y[a:b], t[a:b], p[a:b]


def _chunk(ev, k, chunk=CHUNK):
    return _cut(ev, k * chunk, (k + 1) * chunk)


def _t_end(ev, k, chunk=CHUNK):
    return ev[4] + (k + 1) * chunk


class _HostIngest:
    """oracle/ref_ingest on the host, as a DSEC loader runs it: the script's down-sampler with the change map carried from
    chunk to chunk, then the crop y < H (dsec_data.py:142-143); polarities are the camera's 2p - 1; time is rebased to
    the stream's first raw timestamp."""

    def __init__(self, scale=2, crop=H):
        self.scale, self.crop = scale, crop
        self.cm, self.base = None, None

    def __call__(self, x, y, t, p01):
        from oracle import ref_ingest as R
        if len(t) and self.base is None:
            self.base = int(t[0])
        ev = dict(x=np.asarray(x, np.uint16), y=np.asarray(y, np.uint16), p=(2 * np.asarray(p01, np.int16) - 1).astype(np.int8),
                  t=np.asarray(t, np.int64))
        s = self.scale
        out, self.cm = R.downsample_events(ev, SH, SW, SH // s, SW // s, change_map=self.cm)
        k = out["y"] < self.crop
        tr = out["t"][k] - (self.base if self.base is not None else 0)
        return out["x"][k].astype(np.int32), out["y"][k].astype(np.int32), tr.astype(np.int32), out["p"][k]

    def rebase(self, t_end):
        return int(t_end) - self.base


def _model():
    model, _ = make_model("s", H, W, batch_size=1)
    return model.cuda()


# ---------------------------------------------------------------------------------------------------------------------
def _ingest_call(raw_np, S, max_raw, fx, fy, ow, oh, crop, cmap, max_chunk):
    from dagr_b200 import _lib
    lib = _lib.load()
    raw = torch.from_numpy(raw_np).cuda()
    out = torch.full((4 * S + 4 * S * max_chunk,), -9, dtype=torch.int32, device="cuda")
    _lib.check(lib.dagr_stream_ingest(_lib.ptr(raw), S, max_raw, fx, fy, ow, oh, crop, _lib.ptr(cmap), _lib.ptr(out), max_chunk,
                                      _lib.stream_ptr()), "stream_ingest")
    o = out.cpu().numpy()
    hdr = o[:4 * S].reshape(S, 4)
    rows = [o[4 * S + 4 * int(h[2]):4 * S + 4 * (int(h[2]) + int(h[0]))].reshape(-1, 4) for h in hdr]
    return hdr, rows


def test_ingest_kernel_equals_reference_golden_chunk_by_chunk():
    """the three cases of downsample_golden.npz (the reference's own numba function, change map carried over three chunks)
    through dagr_stream_ingest at S = 1, no crop, +-1 polarities: 640x480 -> 320x240; 64x48 -> 32x24 with a hot-pixel chunk;
    96x48 -> 32x24 (fx = 3, fy = 2)."""
    from dagr_b200.streaming import pack_raw_stage
    g = np.load(GOLD_PATH)
    MR = 6000                                                     # the largest golden chunk
    for case in range(3):
        iw, ih, ow, oh = (int(v) for v in g[f"c{case}_shape"])
        fx, fy = iw // ow, ih // oh
        cmap = torch.zeros((1, oh, ow), dtype=torch.float32, device="cuda")
        raw = np.zeros(4 + 2 * MR, np.int32)
        for k in range(3):
            x, y, p, t = (g[f"c{case}_k{k}_in_{q}"] for q in "xypt")
            pack_raw_stage(raw, [(x, y, t, p)], [-123], MR, planes=[5])
            hdr, rows = _ingest_call(raw, 1, MR, fx, fy, ow, oh, oh, cmap, MR)
            assert hdr[0].tolist() == [len(rows[0]), -123, 0, 5]
            for j, q in enumerate("xytp"):
                assert np.array_equal(rows[0][:, j].astype(np.int64), g[f"c{case}_k{k}_out_{q}"].astype(np.int64)), (case, k, q)
            assert np.array_equal(cmap[0].cpu().numpy(), g[f"c{case}_k{k}_map"]), (case, k)


def test_ingest_kernel_hot_pixel_raw_limit_and_scale_one():
    """S = 2 at the raw limit (16384 events per stream): stream 0 has half its events in one output cell, stream 1 is
    uniform; both equal oracle/ref_ingest (change map carried, crop y < 215) over three chunks.  At fx = fy = 1 the kernel is
    the identity apart from the crop, and so is the reference's arithmetic (every event passes, the map stays 0)."""
    from dagr_b200.streaming import MAX_RAW, pack_raw_stage
    from oracle import ref_ingest as R
    rng = np.random.default_rng(3)
    S, ow, oh = 2, SW // 2, SH // 2
    cmap = torch.zeros((S, oh, ow), dtype=torch.float32, device="cuda")
    maps = [None, None]
    raw = np.zeros(4 * S + 2 * S * MAX_RAW, np.int32)
    for k in range(3):
        chunks = []
        for s in range(S):
            n = MAX_RAW if k != 1 or s == 0 else 5000
            x, y = rng.integers(0, SW, n).astype(np.uint16), rng.integers(0, SH, n).astype(np.uint16)
            if s == 0:
                hot = rng.random(n) < 0.5
                x[hot] = 100 + rng.integers(0, 2, hot.sum()); y[hot] = 50 + rng.integers(0, 2, hot.sum())
            p = (2 * rng.integers(0, 2, n) - 1).astype(np.int8)
            if s == 0 and k == 2:
                p[hot] = 1                                         # a one-signed hot cell passes every fourth event
            t = np.sort(rng.integers(0, 1000, n)).astype(np.int64) + 1000 * k
            chunks.append((x, y, t, p))
        pack_raw_stage(raw, chunks, [7, 8], MAX_RAW)
        hdr, rows = _ingest_call(raw, S, MAX_RAW, 2, 2, ow, oh, H, cmap, MAX_RAW)
        for s, (x, y, t, p) in enumerate(chunks):
            want, maps[s] = R.downsample_events(dict(x=x, y=y, p=p, t=t), SH, SW, oh, ow, change_map=maps[s])
            keep = want["y"] < H
            got = rows[s]
            assert hdr[s].tolist() == [int(keep.sum()), 7 + s, s * MAX_RAW, 0]
            for j, q in enumerate("xytp"):
                assert np.array_equal(got[:, j].astype(np.int64), want[q][keep].astype(np.int64)), (k, s, q)
            assert np.array_equal(cmap[s].cpu().numpy(), maps[s]), (k, s)
    # scale 1: 640x480 cells (over the 2^18 of the sort key, which fx = fy = 1 does not use), crop to 400 rows
    n = 9000
    x, y = rng.integers(0, SW, n).astype(np.uint16), rng.integers(0, SH, n).astype(np.uint16)
    p = rng.integers(0, 2, n).astype(np.int8)
    t = np.sort(rng.integers(0, 5000, n)).astype(np.int64)
    want, wm = R.downsample_events(dict(x=x, y=y, p=2 * p - 1, t=t), SH, SW, SH, SW)
    assert len(want["t"]) == n and not wm.any()                   # the reference's walk at 1:1 is the identity
    cm1 = torch.zeros((1, SH, SW), dtype=torch.float32, device="cuda")
    raw1 = np.zeros(4 + 2 * 16384, np.int32)
    pack_raw_stage(raw1, [(x, y, t, p)], [0], 16384)
    hdr, rows = _ingest_call(raw1, 1, 16384, 1, 1, SW, SH, 400, cm1, 16384)
    k = y < 400
    assert hdr[0, 0] == int(k.sum())
    assert np.array_equal(rows[0], np.stack([x[k], y[k], t[k], 2 * p[k].astype(np.int32) - 1], 1).astype(np.int32))
    assert not cm1.any()


# ---------------------------------------------------------------------------------------------------------------------
def test_raw_streaming_detector_equals_host_ingest_every_step():
    """dagr-s at 320x215 on a raw 640x480 stream, 2 ms chunks, 20 ms window, eager and replayed steps: detections, live
    window and change map equal a plain StreamingDetector fed the host-ingested chunks, after every step."""
    from dagr_b200.streaming import StreamingDetector
    model = _model()
    ev = _raw_stream(1_500_000, seed=5, t0=123_456)
    det = StreamingDetector(model, window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    ref = StreamingDetector(model, window_us=WINDOW, max_chunk=8192, capacity=1 << 15)
    host = _HostIngest()
    window = []
    for k in range(STEPS):
        c = _chunk(ev, k)
        hc = host(*c)
        out = det.push(*c, t_end=_t_end(ev, k))[0]
        want = ref.push(*hc, t_end=host.rebase(_t_end(ev, k)))[0]
        assert _same(out, want), (k, len(out["boxes"]), len(want["boxes"]))
        st, rs = det.window_state, ref.window_state
        assert st.pop("raw") == len(c[2]) and st == rs, (k, st, rs)
        assert st["appended"] == len(hc[2]) and 0 < st["appended"] < len(c[2]) and not st["overflow"]
        window.append(hc)
        pos, feat = det.live_window()
        rpos, rfeat = ref.live_window()
        assert torch.equal(pos, rpos) and torch.equal(feat, rfeat)
        hx, hy, ht, hp = (np.concatenate(a) for a in zip(*window))
        live = ht >= host.rebase(_t_end(ev, k)) - WINDOW
        assert np.array_equal(pos.cpu().numpy(), np.stack([hx, hy, ht], 1)[live]) and np.array_equal(feat.cpu().numpy(), hp[live])
        assert np.array_equal(det.change_map().numpy(), host.cm), k
    assert det.graph is not None and ref.graph is not None


def test_raw_stream_chunking_does_not_matter():
    """the same raw stream fed as 1 ms and as 2 ms chunks (the change map carries across chunk boundaries, as in the script's
    chunked loop) gives the same live window and change map at every common t_end."""
    from dagr_b200.streaming import StreamingDetector
    model = _model()
    ev = _raw_stream(2_000_000, seed=8, kind="uniform", t0=40_000)
    a = StreamingDetector(model, window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    b = StreamingDetector(model, window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    for k in range(STEPS):
        for h in range(2):
            oa = a.push(*_chunk(ev, 2 * k + h, CHUNK // 2), t_end=_t_end(ev, 2 * k + h, CHUNK // 2))[0]
        ob = b.push(*_chunk(ev, k), t_end=_t_end(ev, k))[0]
        pa, fa = a.live_window()
        pb, fb = b.live_window()
        assert torch.equal(pa, pb) and torch.equal(fa, fb), k
        assert _same(oa, ob), k
        assert np.array_equal(a.change_map().numpy(), b.change_map().numpy()), k


def test_raw_multistream_equals_single_camera_detectors():
    """MultiStreamDetector(sensor=...) with three cameras at different rates: camera 1's raw timestamps are above 2^31 us
    (the int64 rebase), camera 2 has empty chunks (as None and as zero-length) and camera 1 is reset mid-stream and handed
    a new stream.  Each camera equals a single-camera raw StreamingDetector bit for bit, and camera 1 its host ingest."""
    from dagr_b200.streaming import MultiStreamDetector, StreamingDetector
    model = _model()
    evs = [_raw_stream(1_500_000, 5), _raw_stream(600_000, 6, "uniform", t0=3_000_000_000),
           _raw_stream(200_000, 7, gap=(14, 19))]
    S, R = len(evs), 12
    fresh = _raw_stream(800_000, 11, "uniform", t0=7_000_000_123)
    det = MultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    refs = [StreamingDetector(model, window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH)) for _ in range(S)]
    plain = StreamingDetector(model, window_us=WINDOW, max_chunk=8192, capacity=1 << 15)
    host = _HostIngest()
    empty_steps = 0
    for k in range(STEPS):
        if k == R:                                                 # camera 1 is handed to another sensor
            det.reset(1)
            refs[1].reset()
            plain.reset()
            evs[1], host = fresh, _HostIngest()
            assert not det.change_map(1).any() and det.change_map(0).any()
        chunks = [_chunk(ev, k) for ev in evs]
        if len(chunks[2][2]) == 0 and k % 2 == 0:
            chunks[2] = None                                       # both forms of "no events this step"
        out = det.push(chunks, [_t_end(ev, k) for ev in evs])
        empty_steps += det.window_state(2)["raw"] == 0
        for s, ev in enumerate(evs):
            want = refs[s].push(*_chunk(ev, k), t_end=_t_end(ev, k))[0]
            assert _same(out[s], want), (k, s, len(out[s]["boxes"]), len(want["boxes"]))
            assert det.window_state(s) == refs[s].window_state, (k, s)
            assert np.array_equal(det.change_map(s).numpy(), refs[s].change_map().numpy()), (k, s)
        hc = host(*chunks[1])
        want = plain.push(*hc, t_end=host.rebase(_t_end(evs[1], k)))[0]
        assert _same(out[1], want), k
        assert torch.equal(det.live_window(1)[0], plain.live_window()[0]), k
    assert empty_steps >= 3 and det.graph is not None


def test_raw_fusion_multistream_equals_host_ingested_chunks():
    """FusionMultiStreamDetector, S = 2, raw mode: every step equals the same detector fed host-ingested chunks (frames at
    the model's resolution, one frame change per camera)."""
    from dagr_b200.streaming import FusionMultiStreamDetector
    from tests.test_fusion_streaming_gpu import _frames
    model, _ = make_model("s", H, W, batch_size=1, use_image=True, img_net="resnet18")
    model.cuda()
    evs = [_raw_stream(1_000_000, 15), _raw_stream(400_000, 16, "uniform", t0=2_500_000_000)]
    S = len(evs)
    frames = [_frames(2, seed=40 + s) for s in range(S)]
    det = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    ref = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=8192, capacity=1 << 15)
    hosts = [_HostIngest() for _ in range(S)]
    for k in range(STEPS):
        for s in range(S):
            if k in (0, 9 + 6 * s):
                i = 0 if k == 0 else 1
                for d in (det, ref):
                    d.set_frame(s, frames[s][i])
                    d.sync_frame(s)
        chunks = [_chunk(ev, k) for ev in evs]
        hcs = [h(*c) for h, c in zip(hosts, chunks)]
        out = det.push(chunks, [_t_end(ev, k) for ev in evs])
        want = ref.push(hcs, [h.rebase(_t_end(ev, k)) for h, ev in zip(hosts, evs)])
        for s in range(S):
            assert _same(out[s], want[s]), (k, s, len(out[s]["boxes"]), len(want[s]["boxes"]))
            st = det.window_state(s)
            assert st.pop("raw") == len(chunks[s][2]) and st == ref.window_state(s), (k, s)
            assert det.frame_state(s) == ref.frame_state(s), (k, s)
    assert len(det.graphs) == 1


def test_raw_chunks_refused_before_any_device_work():
    """over the raw limit, rebased time outside int32, coordinates outside the sensor, polarities of the other convention:
    ValueError, and nothing changed (no launch, same window, same time base); the stream then goes on as if the bad chunk
    had never been submitted."""
    from dagr_b200.streaming import MultiStreamDetector, StreamingDetector
    model = _model()
    ev = _raw_stream(1_500_000, 9, t0=5_000_000)
    det = StreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15, sensor=(SW, SH))
    ref = StreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    host = _HostIngest()
    x, y, t, p = _chunk(ev, 0)
    bad = [((np.zeros(4097, np.uint16),) * 2 + (np.arange(4097) + t[0], np.ones(4097, np.int8)), "max_chunk"),
           ((x[:3], y[:3], np.array([t[0], t[0] + 1, t[0] + (1 << 31)]), p[:3]), "int32"),
           ((np.array([640], np.uint16), y[:1], t[:1], p[:1]), "sensor"),
           ((x[:2], y[:2], t[:2], np.array([-1, 1], np.int8)), "polarities")]
    for k in range(STEPS):
        if k in (0, 7):
            launches, state = det.eng.launches, (None if k == 0 else det.window_state)
            for c, needle in bad:
                with pytest.raises(ValueError, match=needle):
                    det.submit(*c)
            with pytest.raises(ValueError, match="int32"):
                det.submit(*_chunk(ev, k), t_end=_t_end(ev, k) + (1 << 32))
            assert det.eng.launches == launches and det._tbase == ([None] if k == 0 else [int(ev[2][0])])
            if state is not None:
                assert det.window_state == state
        c = _chunk(ev, k)
        out = det.push(*c, t_end=_t_end(ev, k))[0]
        want = ref.push(*host(*c), t_end=host.rebase(_t_end(ev, k)))[0]
        assert _same(out, want), k
    m = MultiStreamDetector(model, streams=2, window_us=WINDOW, max_chunk=4096, capacity=1 << 15, sensor=(SW, SH), p_is_01=False)
    with pytest.raises(ValueError, match="polarities"):
        m.submit([(x[:2], y[:2], t[:2], np.array([0, 1], np.int8)), None])
    assert m._done is None and m._tbase == [None, None]
