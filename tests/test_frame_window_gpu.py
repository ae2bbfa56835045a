"""Interframe windows on live hybrid cameras (since_frame=True): a step of camera s covers [t_cut, t_end) with t_cut =
max(t_us of the frame it reads, t_end - window_us).  After every step, eager and replayed, the detections must equal bit
for bit model(data) at B = 1 over exactly that window with the frame frame_state reports, and SequenceDetector over the same
[t_begin, t_end) with that frame; live_window() must hold exactly the pushed events of the window.  Covered: switches with and
without sync_frame, chunks that straddle a frame's time (their older rows are gone in that same step), a frame later than
t_end left unused, the window_us cap, empty chunks, reset(), TF32 and bf16 image branches, the reference's interframe
windows driven live, S = 3 cameras against one-camera detectors, the raw sensor with raw frames, and the unchanged default."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_fusion_streaming_gpu import _frames, _model, _same, H, W

pytestmark = pytest.mark.gpu

CAP = 30_000                           # window_us: the cap of a window whose frame is older
RATE = 150_000


def _events(seconds, seed, kind="clustered"):
    from dagr_b200.streaming import synth_stream
    return synth_stream(RATE, seconds, W, H, seed=seed, kind=kind)


def _cut(ev, a, b):
    x, y, t, p = ev
    i, j = np.searchsorted(t, [a, b])
    return x[i:j], y[i:j], t[i:j], p[i:j]


def _empty():
    e = np.zeros(0, np.int32)
    return e.astype(np.int16), e.astype(np.int16), e, e.astype(np.int8)


class _Pushed:
    """the chunks a camera's detector was fed since its last reset, on the host."""

    def __init__(self):
        self.parts = []

    def add(self, c):
        self.parts.append(tuple(np.asarray(a) for a in c))

    def reset(self):
        self.parts = []

    def all(self):
        if not self.parts:
            return _empty()
        return tuple(np.concatenate([p[i] for p in self.parts]) for i in range(4))

    def window(self, tb, te):
        x, y, t, p = self.all()
        k = (t >= tb) & (t < te)
        return x[k], y[k], t[k], p[k]


def _dense(model, win, frame):
    """model(data) at B = 1 over the window's events with the frame normalised as format_data does."""
    from dagr_b200.data import EventBatch
    x, y, t, p = win
    n = len(t)
    pos = torch.from_numpy(np.stack([x, y, t], 1).astype(np.int32)).cuda()
    feat = torch.from_numpy(p.astype(np.float32)).cuda()
    d = EventBatch(x=feat.view(-1, 1).clone(), pos=torch.zeros(n, 3, device="cuda"), batch=torch.zeros(n, dtype=torch.long, device="cuda"),
                   width=torch.tensor([W]), height=torch.tensor([H]), time_window=torch.tensor([1_000_000]),
                   pos_denorm=pos, num_graphs=1, dims=(W, H, 1_000_000), image=frame.cuda().float().unsqueeze(0) / 255.0)
    return model(d)[0][0]


def _sequence(model, pushed, tb, te, frame):
    from dagr_b200.sequence import SequenceDetector
    x, y, t, p = pushed.all()
    seq = SequenceDetector(model, window_us=CAP, max_windows=1)
    return seq.detect(dict(x=x, y=y, t=t, p=p), [te], t_begin=[tb], frames=frame.unsqueeze(0), frame_idx=[0])[0]


def _check(det, model, out, frames, pushed, te, cap=CAP, s=None, sequence=True):
    """one camera after one step: t_begin, the live window, model(data) and SequenceDetector."""
    fs = det.frame_state if s is None else det.frame_state(s)
    tb = max(fs["t_us"], te - cap)
    assert fs["t_begin"] == tb, (fs, te)
    win = pushed.window(tb, te)
    pos, feat = det.live_window() if s is None else det.live_window(s)
    assert np.array_equal(pos.cpu().numpy(), np.stack(win[:3], 1).astype(np.int32)), (fs, te, len(pos), len(win[2]))
    assert np.array_equal(feat.cpu().numpy(), win[3].astype(np.float32))
    st = det.window_state if s is None else det.window_state(s)
    assert st["live"] == len(win[2]) and not st["overflow"], st
    frame = frames[fs["frame"]]
    assert _same(out, _dense(model, win, frame)), (fs, te)
    if sequence:
        assert _same(out, _sequence(model, pushed, tb, te, frame)), (fs, te)
    return fs


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_single_camera_window_starts_at_its_frame(precision):
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model()
    model.image_precision = precision
    ev, frames = _events(0.13, seed=11), _frames(5, seed=12)
    det = FusionStreamingDetector(model, window_us=CAP, max_chunk=4096, capacity=1 << 15, since_frame=True)
    with pytest.raises(ValueError, match="t_us"):
        det.set_frame(frames[0])
    pushed = _Pushed()
    CHUNK = 1_000
    sets = {0: (0, 0, True), 50: (1, 50_000, False), 75: (2, 75_400, True), 95: (3, 97_300, True), 110: (4, 110_000, False)}
    steps = 125
    for k in range(steps):
        te = (k + 1) * CHUNK
        if k in sets:
            i, t_us, sync = sets[k]
            assert det.set_frame(frames[i], t_us=t_us) == i
            if sync:
                det.sync_frame()
        if k == 88:
            det.reset()
            pushed.reset()
        c = _empty() if 62 <= k <= 64 else _cut(ev, k * CHUNK, te)
        pushed.add(c)
        out = det.push(*c, t_end=te)[0]
        fs = _check(det, model, out, frames, pushed, te)
        if k == 0 or 75 <= k < 95:
            assert fs["frame"] == (0 if k == 0 else 2) and fs["pending"] is None, (k, fs)
        if k == 75:                                                   # the chunk straddles the frame: its older rows are gone
            older = int(((c[2] >= 75_000) & (c[2] < 75_400)).sum())
            st = det.window_state
            assert older > 0 and st["appended"] == len(c[2]) - older, (older, st)
        if k in (95, 96):                                             # the frame's time is after t_end: not used yet
            assert fs["frame"] == 2 and fs["pending"] == 3, (k, fs)
        if k == 97:
            assert fs["frame"] == 3 and fs["t_begin"] == 97_300, fs
        if 30 <= k < 50:
            assert fs["t_begin"] == te - CAP, (k, fs)                 # the cap: the frame is older than window_us
    assert set(det.graphs) == {0, 1}


def test_interframe_windows_driven_live_equal_one_sequence_call():
    from dagr_b200.sequence import SequenceDetector, interframe_windows
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model()
    frame_t = [10_000, 60_000, 110_000]
    ev, frames = _events(0.17, seed=13), _frames(len(frame_t), seed=14)
    tb, te, fi = interframe_windows(frame_t, steps=10)
    want = SequenceDetector(model, window_us=50_000).detect(dict(zip("xytp", ev)), te, t_begin=tb, frames=torch.stack(frames),
                                                            frame_idx=fi)
    det = FusionStreamingDetector(model, window_us=50_000, max_chunk=4096, capacity=1 << 15, since_frame=True)
    F, last = len(frame_t), 0
    for i in range(F):
        det.set_frame(frames[i], t_us=frame_t[i])
        det.sync_frame()
        for j in range(10):
            q = j * F + i                                             # interframe_windows is offset-major
            end = int(te[q])
            out = det.push(*_cut(ev, last, end), t_end=end)[0]
            last = end
            fs = det.frame_state
            assert fs["frame"] == i and fs["t_begin"] == frame_t[i] and end - fs["t_us"] == int(te[q] - tb[q]), (i, j, fs)
            assert _same(out, want[q]), (i, j, len(out["boxes"]), len(want[q]["boxes"]))


def test_three_cameras_equal_one_camera_detectors():
    from dagr_b200.streaming import FusionMultiStreamDetector, FusionStreamingDetector
    model = _model()
    S, CHUNK, steps, cap = 3, 2_000, 60, 40_000
    evs = [_events(0.12, seed=20 + s) for s in range(S)]
    frames = [_frames(4, seed=30 + s) for s in range(S)]
    kw = dict(window_us=cap, max_chunk=4096, capacity=1 << 15, since_frame=True)
    det = FusionMultiStreamDetector(model, streams=S, **kw)
    refs = [FusionStreamingDetector(model, **kw) for _ in range(S)]
    pushed = [_Pushed() for _ in range(S)]
    # per camera: frame 0 at 0, then frames at an offset of the camera's own every 50 ms, off the chunk grid
    times = [[0] + [o + 50_000 * j for j in range(3) if 0 < o + 50_000 * j < steps * CHUNK] for o in (50_000, 13_300, 26_600)]
    for k in range(steps):
        for s in range(S):
            for i, t_us in enumerate(times[s]):
                if k * CHUNK <= t_us < (k + 1) * CHUNK:
                    assert det.set_frame(s, frames[s][i], t_us=t_us) == refs[s].set_frame(frames[s][i], t_us=t_us) == i
                    det.sync_frame(s)
                    refs[s].sync_frame()
        if k == 30:
            det.reset(1)
            refs[1].reset()
            pushed[1].reset()
        te = [(k + 1) * CHUNK] * S
        chunks = [None if (s == 2 and 20 <= k < 23) else _cut(evs[s], k * CHUNK, te[s]) for s in range(S)]
        out = det.push(chunks, te)
        for s in range(S):
            c = _empty() if chunks[s] is None else chunks[s]
            pushed[s].add(c)
            want = refs[s].push(*c, t_end=te[s])[0]
            assert _same(out[s], want), (k, s)
            assert det.frame_state(s) == refs[s].frame_state and det.window_state(s) == refs[s].window_state, (k, s)
            _check(det, model, out[s], frames[s], pushed[s], te[s], cap=cap, s=s, sequence=False)
    assert len(det.graphs) == 1


def test_raw_sensor_and_raw_frames_equal_host_ingest():
    from dagr_b200.streaming import FusionStreamingDetector
    from tests.test_raw_frames_gpu import SH, SW, _prepared, _sensor_frames
    from tests.test_raw_stream_gpu import CHUNK, STEPS, _HostIngest, _chunk, _raw_stream, _t_end
    model = _model()
    ev, frames = _raw_stream(1_000_000, seed=21, t0=77_000), _sensor_frames(4, seed=2)
    t0, base = ev[4], int(ev[2][0])                                   # the stream's time base: its first raw timestamp
    kw = dict(window_us=CAP, max_chunk=8192, capacity=1 << 15)
    det = FusionStreamingDetector(model, sensor=(SW, SH), raw_frames=True, since_frame=True, **kw)
    ref = FusionStreamingDetector(model, since_frame=True, **kw)
    slide = FusionStreamingDetector(model, sensor=(SW, SH), raw_frames=True, **kw)
    host = _HostIngest()
    sets = {0: (0, t0, True), 7: (1, t0 + 7 * CHUNK + 900, True), 15: (2, t0 + 15 * CHUNK + 300, False),
            22: (3, t0 + 23 * CHUNK + 500, True)}
    for k in range(STEPS):
        if k in sets:
            i, t_raw, sync = sets[k]
            assert det.set_frame(torch.from_numpy(frames[i]), t_us=t_raw) == ref.set_frame(_prepared(frames[i]), t_us=t_raw - base)
            slide.set_frame(torch.from_numpy(frames[i]))
            if sync:
                det.sync_frame()
                ref.sync_frame()
            else:
                torch.cuda.synchronize()                              # both see the trunk finished and take it at the same step
        c = _chunk(ev, k)
        out = det.push(*c, t_end=_t_end(ev, k))[0]
        hc = host(*c)
        want = ref.push(*hc, t_end=host.rebase(_t_end(ev, k)))[0]
        slide.push(*c, t_end=_t_end(ev, k))
        assert _same(out, want), (k, len(out["boxes"]), len(want["boxes"]))
        fs, fr = det.frame_state, ref.frame_state
        assert fs["frame"] == fr["frame"] and fs["t_us"] - base == fr["t_us"] and fs["t_begin"] - base == fr["t_begin"], (k, fs, fr)
        assert fs["t_begin"] == max(fs["t_us"], _t_end(ev, k) - CAP), (k, fs)
        st = det.window_state
        assert {key: v for key, v in st.items() if key != "raw"} == ref.window_state, k
        cmap = det.change_map()
        assert torch.equal(cmap, slide.change_map()) and np.array_equal(cmap.numpy(), host.cm), k
        if k in (22, 23):
            assert fs["frame"] == (2 if k == 22 else 3), (k, fs)
    assert set(det.graphs) == {0, 1}


# ---------------------------------------------------------------------------------------------------------------------
_KERNEL, _MEMCPY, _GRAPH = 0, 1, 5                   # CUgraphNodeType


def _node_types(graph):
    """{node type: count} of a CUDA graph, child graphs included (driver API)."""
    cu = C.CDLL("libcuda.so.1")
    n = C.c_size_t(0)
    assert cu.cuGraphGetNodes(C.c_void_p(graph), None, C.byref(n)) == 0
    nodes = (C.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(C.c_void_p(graph), nodes, C.byref(n)) == 0
    out = {}
    for node in nodes:
        ty = C.c_int(0)
        assert cu.cuGraphNodeGetType(C.c_void_p(node), C.byref(ty)) == 0
        if ty.value == _GRAPH:
            child = C.c_void_p(0)
            assert cu.cuGraphChildGraphNodeGetGraph(C.c_void_p(node), C.byref(child)) == 0
            for k, v in _node_types(child.value).items():
                out[k] = out.get(k, 0) + v
        else:
            out[ty.value] = out.get(ty.value, 0) + 1
    return out


def _captured_step(det):
    """the node types of the detector's step as its own capture records it (kept, not replayed)."""
    g = torch.cuda.CUDAGraph(keep_graph=True)
    saved = det.ctl.clone()
    det.stream.synchronize()
    with torch.cuda.stream(det.stream):
        with torch.cuda.graph(g, stream=det.stream):
            det._enqueue()
    det.ctl.copy_(saved)
    return _node_types(g.raw_cuda_graph())


def test_default_keeps_the_stage_and_the_captured_step():
    from dagr_b200.streaming import FusionMultiStreamDetector, FusionStreamingDetector
    model = _model()
    ev, frames = _events(0.01, seed=40), _frames(1, seed=41)
    kw = dict(window_us=CAP, max_chunk=4096, capacity=1 << 15)
    for make in (lambda **o: FusionStreamingDetector(model, **kw, **o), lambda **o: FusionMultiStreamDetector(model, streams=2, **kw, **o)):
        dets = [make(), make(since_frame=False), make(since_frame=True)]
        for k in range(3):
            for d in dets:
                c = _cut(ev, k * 1_000, (k + 1) * 1_000)
                if isinstance(d, FusionMultiStreamDetector):
                    for s in range(2):
                        if k == 0:
                            d.set_frame(s, frames[0], t_us=0)
                    d.push([c, None], [(k + 1) * 1_000] * 2)
                else:
                    if k == 0:
                        d.set_frame(frames[0], t_us=0)
                    d.push(*c, t_end=(k + 1) * 1_000)
        plain, off, on = dets
        n, S = plain.stage_bytes // 4, plain.S
        assert off.stage_bytes == plain.stage_bytes and np.array_equal(off._stage_np, plain._stage_np)
        # since_frame: the same chunk layout (its cuts start at the frame), then the cut stage with those cuts
        assert on.stage_bytes == 4 * (on._cut_off + 8 * S) and np.array_equal(on._stage_np[4 * S:n], plain._stage_np[4 * S:])
        hdr = on._stage_np[:4 * S].reshape(S, 4)
        assert on._stage_np[on._cut_off:on._cut_off + 4 * S].reshape(S, 4).tolist() == [[0, int(h[1]), 0, int(h[3])] for h in hdr]
        assert len(plain.graphs) == len(off.graphs) == len(on.graphs) == 1
        a, b, c = (_captured_step(d) for d in dets)
        assert a == b, (a, b)
        assert c[_KERNEL] == a[_KERNEL] + 2 and c.get(_MEMCPY, 0) == a.get(_MEMCPY, 0) + 1, (a, c)
