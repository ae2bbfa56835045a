"""Raw camera frames on the device: dagr_frame_preprocess must equal the reference's own frame preparation
(DSEC.preprocess_image, dsec_data.py:149-154, with the real OpenCV; golden vectors) byte for byte, and its f32 form the
`.float() / 255.0` of that u8 image bit for bit.  A fusion detector with raw_frames=True, fed a 640x480 camera's frames,
must equal bit for bit the same detector fed frames prepared on the host by oracle/ref_frame (which equals the golden
vectors), after every step: eager and replayed, both slots, with and without sync_frame, two frames in a row, a frame change
on an empty chunk, per camera with several cameras and a per-camera reset, and after refused frames."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests.helpers import make_model
from tests.test_fusion_streaming_gpu import _same
from tests.test_raw_stream_gpu import STEPS, _chunk, _raw_stream, _t_end

pytestmark = pytest.mark.gpu

SW, SH, W, H, SCALE = 640, 480, 320, 215, 2
WINDOW = 20_000
GOLD_PATH = Path(__file__).resolve().parent / "golden" / "frame_golden.npz"


def _model():
    model, _ = make_model("s", H, W, batch_size=1, use_image=True, img_net="resnet18")
    return model.cuda()


def _sensor_frames(n, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (SH, SW, 3), dtype=np.uint8) for _ in range(n)]


def _prepared(frame):
    """the model-resolution frame a host-side loader hands the detector: u8 [3, H, W]."""
    from oracle.ref_frame import preprocess_image
    return torch.from_numpy(preprocess_image(frame, H, W, SCALE)[0])


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------
def test_frame_kernel_equals_reference_golden_both_outputs():
    from dagr_b200 import ingest
    g = np.load(GOLD_PATH)
    lut = ingest.frame_lut("cuda")
    for i in range(int(g["cases"])):
        h, w, s = (int(v) for v in g[f"c{i}_geom"])
        src = torch.from_numpy(g[f"c{i}_in"]).cuda().unsqueeze(0)
        want = torch.from_numpy(g[f"c{i}_out"]).cuda()
        u8 = ingest.preprocess_frames(src, h, w, s)
        assert u8.dtype == torch.uint8 and torch.equal(u8, want), (i, int((u8 != want).sum()))
        f32 = ingest.preprocess_frames(src, h, w, s, lut)
        assert f32.dtype == torch.float32 and torch.equal(_bits(f32), _bits(want.float() / 255.0)), i


def test_preprocess_image_batch_equals_per_frame_golden():
    from dagr_b200 import ingest
    g = np.load(GOLD_PATH)
    order = [0, 1, 1, 0]                                              # the two 640x480 cases
    batch = torch.from_numpy(np.stack([g[f"c{i}_in"] for i in order])).cuda()
    out = ingest.preprocess_image(batch, H, W, SCALE)
    assert out.shape == (4, 3, H, W) and out.dtype == torch.uint8
    for j, i in enumerate(order):
        assert torch.equal(out[j].cpu(), torch.from_numpy(g[f"c{i}_out"][0])), j
    one = ingest.preprocess_image(batch[1], H, W, SCALE)              # [sh, sw, 3] -> [1, 3, H, W]
    assert torch.equal(one.cpu(), torch.from_numpy(g["c1_out"]))
    wide = torch.zeros((SH, SW + 8, 3), dtype=torch.uint8, device="cuda")
    wide[:, :SW] = batch[0]
    assert torch.equal(ingest.preprocess_image(wide[:, :SW], H, W, SCALE).cpu(), torch.from_numpy(g["c0_out"]))   # strided
    with pytest.raises(RuntimeError, match="src_w"):
        ingest.preprocess_image(batch[:, :, :SW - 2], H, W, SCALE)


# ---------------------------------------------------------------------------------------------------------------------
def _set(det, ref, frame, cam=None, device=False, sync=True):
    """the same frame to both detectors: raw to `det`, prepared on the host to `ref`; host or device tensors.  Unsynced
    frames are left to the steps' own promotion (a non-blocking event query); the device is drained first so that both
    detectors see the trunk finished and promote at the same step."""
    raw, prep = torch.from_numpy(frame), _prepared(frame)
    if device:
        raw, prep = raw.cuda(), prep.cuda()
    args = () if cam is None else (cam,)
    fid = det.set_frame(*args, raw)
    assert ref.set_frame(*args, prep) == fid
    if sync:
        det.sync_frame(*args)
        ref.sync_frame(*args)
    else:
        torch.cuda.synchronize()
    return fid


def test_raw_frames_streaming_detector_equals_host_prepared_frames():
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model()
    ev, frames = _raw_stream(1_000_000, seed=21, t0=77_000), _sensor_frames(4, seed=1)
    kw = dict(window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    det = FusionStreamingDetector(model, raw_frames=True, **kw)
    ref = FusionStreamingDetector(model, **kw)
    for k in range(STEPS):
        if k == 0:
            _set(det, ref, frames[0])                                 # host frame, synced: slot 0
        elif k == 6:
            _set(det, ref, frames[1], device=True, sync=False)        # device frame, promoted by the step: slot 1
        elif k == 12:
            _set(det, ref, frames[2], sync=False)
        elif k == 18:                                                 # two frames in a row: the first is waited for
            _set(det, ref, frames[3], device=True, sync=False)
            _set(det, ref, frames[0])
        elif k == 24:                                                 # a frame change on an empty chunk
            _set(det, ref, frames[1])
            e = np.zeros(0, np.int64)
            out = det.push(e.astype(np.uint16), e.astype(np.uint16), e, e.astype(np.int8), t_end=_t_end(ev, k - 1))[0]
            want = ref.push(e.astype(np.uint16), e.astype(np.uint16), e, e.astype(np.int8), t_end=_t_end(ev, k - 1))[0]
            assert _same(out, want) and det.frame_state == ref.frame_state == dict(frame=5, t_us=None, pending=None)
            assert det.window_state["appended"] == 0 and det.window_state == ref.window_state
        c = _chunk(ev, k)
        out = det.push(*c, t_end=_t_end(ev, k))[0]
        want = ref.push(*c, t_end=_t_end(ev, k))[0]
        assert _same(out, want), (k, len(out["boxes"]), len(want["boxes"]))
        assert det.frame_state == ref.frame_state, (k, det.frame_state, ref.frame_state)
        assert det.window_state == ref.window_state, k
        if k in (1, 7, 13):
            assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(det._frames.frame(det._cur)[0], ref._frames.frame(ref._cur)[0])), k
    assert set(det.graphs) == {0, 1} and det.frame_state["frame"] == 5


def test_raw_frames_multistream_per_camera_equals_host_prepared_frames():
    from dagr_b200.streaming import FusionMultiStreamDetector
    model = _model()
    evs = [_raw_stream(1_000_000, 31), _raw_stream(500_000, 32, "uniform", t0=2_600_000_000), _raw_stream(300_000, 33)]
    S = len(evs)
    frames = [_sensor_frames(3, seed=50 + s) for s in range(S)]
    kw = dict(window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    det = FusionMultiStreamDetector(model, streams=S, raw_frames=True, **kw)
    ref = FusionMultiStreamDetector(model, streams=S, **kw)
    at = {0: [(0, 0, True), (1, 0, True), (2, 0, True)], 4: [(1, 1, False)], 7: [(0, 1, True), (2, 1, False)],
          12: [(2, 2, True)], 15: [(1, 2, False), (0, 2, False)], 22: [(1, 0, True)]}    # step: (camera, frame, synced)
    for k in range(STEPS):
        if k == 10:
            det.reset(1)
            ref.reset(1)
        for s, i, sync in at.get(k, []):
            _set(det, ref, frames[s][i], cam=s, device=(s + i) % 2 == 1, sync=sync)
        chunks = [_chunk(ev, k) for ev in evs]
        t_end = [_t_end(ev, k) for ev in evs]
        out = det.push(chunks, t_end)
        want = ref.push(chunks, t_end)
        for s in range(S):
            assert _same(out[s], want[s]), (k, s, len(out[s]["boxes"]), len(want[s]["boxes"]))
            assert det.frame_state(s) == ref.frame_state(s), (k, s)
            assert det.window_state(s) == ref.window_state(s), (k, s)
    assert len(det.graphs) == 1 and [det.frame_state(s)["frame"] for s in range(S)] == [2, 3, 2]


def test_refused_raw_frames_leave_no_trace():
    from dagr_b200.streaming import FusionMultiStreamDetector, FusionStreamingDetector
    model = _model()
    ev, frames = _raw_stream(1_000_000, seed=41), _sensor_frames(2, seed=2)
    kw = dict(window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    det = FusionStreamingDetector(model, raw_frames=True, **kw)
    ref = FusionStreamingDetector(model, **kw)
    bad = [(np.zeros((H, W, 3), np.uint8), "480, 640, 3"), (np.zeros((3, SH, SW), np.uint8), "480, 640, 3"),
           (np.zeros((1, SH, SW, 3), np.uint8), "480, 640, 3"), (np.zeros((SH, SW, 3), np.float32), "uint8"),
           (torch.zeros((SH, SW, 4), dtype=torch.uint8, device="cuda"), "480, 640, 3"),
           (torch.zeros((SH - 1, SW, 3), dtype=torch.uint8, device="cuda"), "480, 640, 3")]
    for k in range(STEPS):
        if k in (0, 9):
            launches, state = det.eng.launches, det._cam.state()
            for img, needle in bad:
                with pytest.raises(ValueError, match=needle):
                    det.set_frame(img)
            assert det.eng.launches == launches and det._cam.nframes == k // 9 and det._cam.state() == state
            assert det._cam.pending is None
            _set(det, ref, frames[k // 9], sync=k == 0)
        c = _chunk(ev, k)
        out = det.push(*c, t_end=_t_end(ev, k))[0]
        want = ref.push(*c, t_end=_t_end(ev, k))[0]
        assert _same(out, want), k
        assert det.frame_state == ref.frame_state, k
    m = FusionMultiStreamDetector(model, streams=2, raw_frames=True, **kw)
    with pytest.raises(ValueError, match="480, 640, 3"):
        m.set_frame(0, frames[0][:, :, :2])
    assert m._cams[0].nframes == 0 and m._cams[0].pending is None and m._frames.feats is None
