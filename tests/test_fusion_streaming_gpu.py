"""FusionStreamingDetector: the hybrid (image + events) model streamed with one CUDA graph replay per chunk and one trunk
run per frame.  After every checked step the detections must equal, bit for bit, the synchronous forward model(data) over
the live window with the image of the frame the step reports -- across eager and replayed steps, both frame slots, frames
switched with and without sync_frame(), a frame change on an empty chunk, a reset and two set_frame calls in a row."""
import numpy as np
import pytest
import torch

from tests.helpers import make_model

pytestmark = pytest.mark.gpu

W, H = 320, 215
WINDOW, CHUNK, STEPS = 20_000, 2_000, 30
CHECKS = (0, 1, 2, 5, 10, 11, 12, 16, 20, 21, 29)      # eager (0, 1, and 10: slot 1's first step) and replayed steps, both slots
FRAMES_AT = (0, 10, 20)                                  # synced frames: slot 0, slot 1, slot 0 again


def _model():
    model, _ = make_model("s", H, W, batch_size=1, use_image=True, img_net="resnet18")
    return model.cuda()


def _frames(n, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8) for _ in range(n)]


def _stream(rate=300_000, seed=5, kind="clustered"):
    from dagr_b200.streaming import synth_stream
    return synth_stream(rate, STEPS * CHUNK * 1e-6, W, H, seed=seed, kind=kind)


def _chunk(ev, k):
    x, y, t, p = ev
    a, b = np.searchsorted(t, [k * CHUNK, (k + 1) * CHUNK])
    return x[a:b], y[a:b], t[a:b], p[a:b]


def _same(a, b):
    return (len(a["boxes"]) == len(b["boxes"]) and torch.equal(a["boxes"], b["boxes"].cpu()) and torch.equal(a["scores"], b["scores"].cpu())
            and torch.equal(a["labels"], b["labels"].cpu()))


def _dense(model, pos, feat, frame):
    """the synchronous forward over one live window with the frame's image normalised as format_data does (on the device,
    like the detector)."""
    from dagr_b200.data import EventBatch
    n = len(feat)
    d = EventBatch(x=feat.view(-1, 1).clone(), pos=torch.zeros(n, 3, device="cuda"), batch=torch.zeros(n, dtype=torch.long, device="cuda"),
                   width=torch.tensor([W]), height=torch.tensor([H]), time_window=torch.tensor([1_000_000]),
                   pos_denorm=pos.clone(), num_graphs=1, dims=(W, H, 1_000_000), image=frame.cuda().float().unsqueeze(0) / 255.0)
    return model(d)[0][0]


def _check(det, model, out, frames):
    fs = det.frame_state
    pos, feat = det.live_window()
    want = _dense(model, pos, feat, frames[fs["frame"]])
    assert _same(out, want), (fs, len(out["boxes"]), len(want["boxes"]))
    return fs


def test_fusion_stream_equals_dense_forward_with_its_frame():
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model()
    ev, frames = _stream(), _frames(len(FRAMES_AT))
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    fid = -1
    for k in range(STEPS):
        if k in FRAMES_AT:
            fid = det.set_frame(frames[FRAMES_AT.index(k)], t_us=k * CHUNK)
            assert fid == FRAMES_AT.index(k)
            det.sync_frame()
        out = det.push(*_chunk(ev, k), (k + 1) * CHUNK)[0]
        if k not in CHECKS:
            continue
        t, te = ev[2], (k + 1) * CHUNK
        live = (t >= te - WINDOW) & (t < te)
        st = det.window_state
        assert st["live"] == int(live.sum()) and not st["overflow"], (k, st)
        pos, feat = det.live_window()
        assert np.array_equal(pos[:, 2].cpu().numpy(), t[live])
        fs = _check(det, model, out, frames)
        assert fs == dict(frame=fid, t_us=FRAMES_AT[fid] * CHUNK, pending=None), (k, fs)
        # the slot holds exactly what the branch computes for this frame (the dense forward above just ran it)
        feats, outs = det._slots[det._cur]
        assert all(torch.equal(a, b) for a, b in zip(feats, model.last_image_feats))
        assert all(torch.equal(a, b) for key in outs for a, b in zip(outs[key], model.last_image_outs[key]))
    assert set(det.graphs) == {0, 1} and all(g is not None for g in det.graphs.values())


def test_fusion_stream_switches_frames_without_blocking():
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model()
    ev, frames = _stream(seed=6, kind="uniform"), _frames(4, seed=4)
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    det.set_frame(frames[0])
    seen, last = [], 0
    for k in range(STEPS):
        if k in (6, 12, 13):                              # 13: a second frame while 12's may still be pending
            det.set_frame(frames[(6, 12, 13).index(k) + 1])
        if k == 24:
            det.sync_frame()
        out = det.push(*_chunk(ev, k), (k + 1) * CHUNK)[0]
        fs = _check(det, model, out, frames)
        assert fs["frame"] >= last, (k, fs)
        last = fs["frame"]
        seen.append(fs["frame"])
        if k >= 24:
            assert fs["frame"] == 3 and fs["pending"] is None, (k, fs)
    assert seen[0] == 0 and 3 in seen


def test_fusion_stream_frame_change_alone_changes_the_output():
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model()
    ev, frames = _stream(seed=7), _frames(2, seed=5)
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    det.set_frame(frames[0])
    for k in range(15):
        prev = det.push(*_chunk(ev, k), (k + 1) * CHUNK)[0]
    pos0, feat0 = det.live_window()
    det.set_frame(frames[1])
    det.sync_frame()
    e = np.zeros(0, np.int32)
    out = det.push(e, e, e, e, 15 * CHUNK)[0]              # no events, same t_end: the window stays as it is
    st = det.window_state
    assert st["appended"] == 0 and st["evicted"] == 0
    pos1, feat1 = det.live_window()
    assert torch.equal(pos0, pos1) and torch.equal(feat0, feat1)
    assert det.frame_state["frame"] == 1
    _check(det, model, out, frames)
    assert not _same(prev, _dense(model, pos1, feat1, frames[1]))


def test_fusion_stream_reset_keeps_the_frame_and_set_frame_twice():
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model()
    ev, frames = _stream(seed=8), _frames(4, seed=6)
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    det.set_frame(frames[0])
    for k in range(12):
        det.push(*_chunk(ev, k), (k + 1) * CHUNK)
    det.reset()
    c = _chunk(ev, 12)
    out = det.push(*c, 13 * CHUNK)[0]
    assert det.window_state["live"] == len(c[2]) and det.frame_state["frame"] == 0
    _check(det, model, out, frames)
    # a step in flight reads the current slot while two frames arrive: the first is promoted, the second's copy goes into
    # the slot that step reads and must wait for it
    det.submit(*_chunk(ev, 13), 14 * CHUNK)
    assert det.set_frame(frames[1]) == 1
    assert det.set_frame(frames[2]) == 2
    out = det.result()[0]
    assert _check(det, model, out, frames)["frame"] == 0
    out = det.push(*_chunk(ev, 14), 15 * CHUNK)[0]
    assert _check(det, model, out, frames)["frame"] in (1, 2)
    det.sync_frame()
    for k in (15, 16):
        out = det.push(*_chunk(ev, k), (k + 1) * CHUNK)[0]
        assert _check(det, model, out, frames)["frame"] == 2
