"""InterframeEvaluation end to end: ev.compute() equals, float for float, one DetectionBuffer per offset fed per-window
dicts built from the oracle's labels (oracle/ref_labels.py, NumPy-1 rule) and SequenceDetector's detections, over two
recordings added in order, on events-only and hybrid models and with raw sensor events and camera frames.  The single
grouped evaluate launch gives the precision slices of G separate launches, reference_batch_size drops exactly the trailing
pairs of the dataset, and ev.detections() equals records_from_device of the same windows."""
import numpy as np
import pytest
import torch

from dagr_b200 import evaluation
from dagr_b200.evaluation import DetectionBuffer
from dagr_b200.interframe import InterframeEvaluation
from dagr_b200.sequence import SequenceDetector, interframe_windows
from dagr_b200.utils.buffers import records_from_device
from oracle import ref_labels as R
from tests import interframe_cases as IC
from tests.helpers import make_model

pytestmark = pytest.mark.gpu

W, H = 320, 215
SW, SH = 640, 480
STEPS, MIN_H, MIN_D = 5, 10, 15


@pytest.fixture(scope="module")
def model():
    return make_model("s", H, W, batch_size=1)[0].cuda()


@pytest.fixture(scope="module")
def hybrid():
    return make_model("s", H, W, batch_size=1, use_image=True, img_net="resnet18")[0].cuda()


def _frames(n, shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n,) + shape, generator=g, dtype=torch.uint8)


def recordings(use_image, sensor=None, raw_frames=False):
    out = []
    for k, (seconds, seed) in enumerate(((0.9, 21), (0.45, 22))):
        ev, ft, tracks = IC.recording(seconds, seed, W, H, sensor=sensor, t0=0 if sensor is None else 3_000_000_000 + k * 10**7)
        frames = None
        if use_image:
            frames = _frames(len(ft), (SH, SW, 3) if raw_frames else (3, H, W), seed)
        out.append((f"seq_{k}", ev, frames, ft, tracks))
    return out


def user_route(model, recs, offsets, sensor=None, raw_frames=False, max_pairs=None):
    """what a user does today: the oracle's labels, one dict per window, SequenceDetector's detections, one DetectionBuffer
    per offset.  -> ({n_us: metrics}, per-recording (pairs, det, ndet, t_end))"""
    bufs = {n_us: DetectionBuffer(H, W, list(R.CLASSES)) for n_us in offsets}
    left = max_pairs
    runs = []
    per_offset = {n_us: ([], []) for n_us in offsets}
    for name, ev, frames, ft, tracks in recs:
        pairs, lab = R.recording_labels(tracks, ft, IC.SOURCE, W, H, 2, MIN_H, MIN_D)
        if left is not None:
            pairs, lab = pairs[:left], lab[:left]
            left -= len(pairs)
        if not len(pairs):
            continue
        tb, te, fi = interframe_windows(ft[pairs[:, 0]], STEPS, 50_000)
        det = SequenceDetector(model, sensor=sensor, raw_frames=raw_frames)
        kw = dict(frames=frames, frame_idx=pairs[fi, 0]) if frames is not None else {}
        dets = det.detect(ev, te, t_begin=tb, **kw)
        runs.append((name, pairs, det.last, te))
        P = len(pairs)
        for g, n_us in enumerate(offsets):
            for p, (d0, d1) in enumerate(lab):
                b, lb = R.window_targets(d0, d1, int(ft[pairs[p, 0]]) + n_us, W, H, MIN_H, MIN_D, "numpy1")
                per_offset[n_us][0].append(dets[g * P + p])
                per_offset[n_us][1].append(dict(boxes=torch.from_numpy(b), labels=torch.from_numpy(lb)))
    out = {}
    for n_us in offsets:
        bufs[n_us].update(*per_offset[n_us], "dsec")
        out[n_us] = bufs[n_us].compute()
    return out, runs


def same_metrics(got, want):
    assert list(got) == list(want)
    for n_us in want:
        assert got[n_us] == want[n_us], (n_us, got[n_us], want[n_us])          # float for float


def evaluation_for(model, recs, **kw):
    ev = InterframeEvaluation(model, IC.SOURCE, steps=STEPS, min_bbox_height=MIN_H, min_bbox_diag=MIN_D, **kw)
    for name, events, frames, ft, tracks in recs:
        ev.add(events, frames, ft, tracks, sequence=name)
    return ev


def test_events_only_equals_one_buffer_per_offset(model):
    recs = recordings(False)
    ev = evaluation_for(model, recs)
    got = ev.compute()
    want, _ = user_route(model, recs, ev.offsets)
    same_metrics(got, want)
    assert any(m["mAP"] > 0 for m in got.values())
    assert all(r["P"] > 3 for r in ev.recordings)


@pytest.mark.parametrize("raw", [False, True])
def test_hybrid_equals_one_buffer_per_offset(hybrid, raw):
    kw = dict(sensor=(SW, SH), raw_frames=True) if raw else {}
    recs = recordings(True, **kw)
    ev = evaluation_for(hybrid, recs, **kw)
    got = ev.compute()
    want, _ = user_route(hybrid, recs, ev.offsets, **kw)
    same_metrics(got, want)
    assert any(m["mAP"] > 0 for m in got.values())


def test_grouped_launch_equals_one_launch_per_offset(model):
    recs = recordings(False)
    ev = evaluation_for(model, recs)
    ev.compute()
    precision = ev.last[0].cpu().numpy()
    K, compared = ev.K, 0
    for g in range(ev.steps):
        gts, dts = [], []
        for r in ev.recordings:
            go, do = r["gt_off"].cpu().numpy(), r["dt_off"].cpu().numpy()
            for q in range(g * r["P"], (g + 1) * r["P"]):
                gts.append(dict(boxes=r["gt_box"][go[q]:go[q + 1]], labels=r["gt_label"][go[q]:go[q + 1]] - g * K))
                dts.append(dict(boxes=r["dt_box"][do[q]:do[q + 1]], scores=r["dt_score"][do[q]:do[q + 1]],
                                labels=r["dt_label"][do[q]:do[q + 1]] - g * K))
        out = evaluation.accumulate(gts, dts, K)                                # one launch for this offset alone
        if out is None:
            continue
        one = out[0].cpu().numpy()
        assert np.array_equal(one.view(np.int64), precision[:, :, g * K:(g + 1) * K].view(np.int64)), g
        compared += 1
    assert compared >= ev.steps - 1


def test_reference_batch_size_drops_the_trailing_pairs(model):
    recs = recordings(False)
    full = evaluation_for(model, recs)
    P = [r["P"] for r in full.recordings]
    total, drop = sum(P), P[1] + 2                                              # the drop reaches into the first recording
    b = total - drop
    assert b > drop and total % b == drop
    ev = evaluation_for(model, recs, reference_batch_size=b)
    got = ev.compute()
    want, runs = user_route(model, recs, ev.offsets, max_pairs=total - drop)
    same_metrics(got, want)
    assert [r["kept"] for r in ev.recordings] == [P[0] - 2, 0]
    d = ev.detections()
    assert list(d) == ["seq_0"]                                                 # seq_1 is dropped whole
    assert len(d["seq_0"]) == sum(int(n) for n in runs[0][2][1].cpu().numpy())


def test_detections_equal_records_of_the_same_windows(model):
    recs = recordings(False)
    ev = evaluation_for(model, recs)
    got = ev.detections()
    _, runs = user_route(model, recs, ev.offsets)
    for name, pairs, (det, ndet), te in runs:
        recs_w = records_from_device(det, ndet, te.tolist())
        want = np.concatenate(recs_w)
        want = want[np.argsort(want["t"], kind="stable")]
        assert got[name].dtype == want.dtype and got[name].tobytes() == want.tobytes(), name
        assert len(want) > 0


def test_bad_input_raises_before_device_work(model, hybrid):
    recs = recordings(False)
    name, events, _, ft, tracks = recs[0]
    ev = InterframeEvaluation(model, IC.SOURCE, steps=STEPS)
    with pytest.raises(ValueError):
        ev.add(events, _frames(len(ft), (3, H, W), 0), ft, tracks, sequence=name)
    with pytest.raises(ValueError):
        InterframeEvaluation(hybrid, IC.SOURCE).add(events, None, ft, tracks, sequence=name)
    with pytest.raises(ValueError):
        ev.add(events, None, ft, tracks[::-1], sequence=name)
    with pytest.raises(KeyError):
        InterframeEvaluation(model, ("car", "boat"))
    assert ev.recordings == [] and all(m["mAP"] == 0.0 for m in ev.compute().values())
