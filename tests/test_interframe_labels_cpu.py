"""The interframe evaluation's label chain on the host: oracle/ref_labels.py and dagr_b200/labels.py against
tests/golden/interframe_labels_golden.npz, which holds the reference's own results (filter_tracks, preprocess_detections,
interpolate_tracks under both promotion rules, the test-time Crop and filter_small_bboxes; made by
tests/golden/make_interframe_labels_golden.py).  The fixture's recordings hold pairs that are not consecutive, a track-id
mismatch, IoU one float32 step either side of 0.10, classes mapped to None, boxes across every border and one clamped to
zero width, size filters one ulp either side, a frame without labels, and offsets with r = 0, r = 1, r in between and
r > 1."""
from pathlib import Path

import numpy as np
import pytest

from dagr_b200 import labels as L
from oracle import ref_labels as R

Z = np.load(Path(__file__).parent / "golden" / "interframe_labels_golden.npz")
NAMES = ("rec_a", "rec_b")
SOURCE = tuple(str(s) for s in Z["source"])
W, H, SCALE, MIN_H, MIN_D = (int(v) for v in Z["dims"])
OFFSETS = [int(v) for v in Z["offsets"]]


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32 if a.dtype == np.float32 else a.dtype)


def same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(bits(a), bits(b))


def rec(name):
    return Z[f"{name}_tracks"], Z[f"{name}_image_ts"]


def oracle_targets(name, rule):
    tracks, ts = rec(name)
    pairs, frames = R.recording_labels(tracks, ts, SOURCE, W, H, SCALE, MIN_H, MIN_D)
    boxes, labels, off = [], [], [0]
    for n_us in OFFSETS:
        for (i0, _), (d0, d1) in zip(pairs, frames):
            b, lab = R.window_targets(d0, d1, int(ts[i0]) + n_us, W, H, MIN_H, MIN_D, rule)
            boxes.append(b)
            labels.append(lab)
            off.append(off[-1] + len(b))
    return np.concatenate(boxes).reshape(-1, 4), np.concatenate(labels), np.array(off, np.int64)


@pytest.mark.parametrize("name", NAMES)
def test_fixture_covers_its_cases(name):
    assert Z[f"{name}_pairs"].tolist() == [[0, 1], [1, 2], [8, 9], [10, 11], [12, 13]]   # 3 empty, 4/5 ids, 6/7 IoU, 13/14
    assert not same(Z[f"{name}_numpy1_box"], Z[f"{name}_nep50_box"])                     # the two rules differ
    tid = Z[f"{name}_tid0"]
    assert 18 in tid and 19 not in tid and 20 in tid and 21 not in tid and 16 not in tid and 17 not in tid and 40 not in tid


@pytest.mark.parametrize("name", NAMES)
def test_oracle_pairs_and_tables_equal_the_reference(name):
    tracks, ts = rec(name)
    pairs, frames = R.recording_labels(tracks, ts, SOURCE, W, H, SCALE, MIN_H, MIN_D)
    assert np.array_equal(pairs, Z[f"{name}_pairs"])
    off = Z[f"{name}_off"]
    for j in (0, 1):
        rows = np.concatenate([f[j] for f in frames])
        assert same(np.stack([rows[k] for k in "xywh"], 1).astype(np.float32), Z[f"{name}_box{j}"])
        assert np.array_equal(rows["class_id"].astype(np.int64), Z[f"{name}_cls{j}"])
        assert np.array_equal(rows["track_id"].astype(np.int64), Z[f"{name}_tid{j}"])
    assert np.array_equal(np.cumsum([0] + [len(f[0]) for f in frames]), off)


@pytest.mark.parametrize("rule", R.RULES)
@pytest.mark.parametrize("name", NAMES)
def test_oracle_window_targets_equal_the_reference(name, rule):
    box, lab, off = oracle_targets(name, rule)
    assert same(box, Z[f"{name}_{rule}_box"])
    assert np.array_equal(lab, Z[f"{name}_{rule}_label"]) and np.array_equal(off, Z[f"{name}_{rule}_off"])


@pytest.mark.parametrize("name", NAMES)
def test_product_pair_labels_equal_the_reference(name):
    tracks, ts = rec(name)
    pl = L.pair_labels(tracks, ts, SOURCE, W, H, SCALE, MIN_H, MIN_D)
    assert np.array_equal(pl.pairs, Z[f"{name}_pairs"])
    assert np.array_equal(pl.t, ts[pl.pairs])
    assert np.array_equal(pl.off, Z[f"{name}_off"])
    assert same(pl.box0, Z[f"{name}_box0"]) and same(pl.box1, Z[f"{name}_box1"])
    assert np.array_equal(pl.cls, Z[f"{name}_cls0"]) and np.array_equal(pl.track_id, Z[f"{name}_tid0"])
    assert np.array_equal(pl.track_id, Z[f"{name}_tid1"])


@pytest.mark.parametrize("rule", R.RULES)
@pytest.mark.parametrize("name", NAMES)
def test_r_zero_and_one_give_the_frame_labels(name, rule):
    tracks, ts = rec(name)
    pairs, frames = R.recording_labels(tracks, ts, SOURCE, W, H, SCALE, MIN_H, MIN_D)
    ones = 0
    for (i0, i1), (d0, d1) in zip(pairs, frames):
        for n_us, want in ((0, d0), (int(ts[i1] - ts[i0]), d1)):
            got = R.window_targets(d0, d1, int(ts[i0]) + n_us, W, H, MIN_H, MIN_D, rule)
            ref = R.test_time_targets(want, W, H, MIN_H, MIN_D)
            assert same(got[0], ref[0]), (name, i0, n_us)
        ones += int(ts[i1] - ts[i0]) in OFFSETS
    assert ones > 0                                                           # the fixture itself has r = 1 windows


def _random_recording(seed, frames=40):
    """many tracks with births, deaths, jumps (IoU drops), class changes to dropped classes and gaps without labels"""
    rng = np.random.default_rng(seed)
    ts = 1_000_000 + np.cumsum(rng.choice([50_000, 50_000, 50_000, 49_000], frames)).astype(np.int64)
    rows = []
    alive = {}
    for f in range(frames):
        if rng.random() < 0.08:
            continue                                                          # a frame without labels
        for tid in list(alive):
            if rng.random() < 0.05:
                del alive[tid]
        while len(alive) < 8:
            alive[int(rng.integers(0, 1 << 20))] = [rng.uniform(-80, 640), rng.uniform(-80, 480), rng.uniform(5, 200),
                                                    rng.uniform(5, 150), int(rng.integers(0, 8))]
        for tid, b in alive.items():
            b[0] += rng.normal(0, 8 if rng.random() > 0.03 else 200)
            b[1] += rng.normal(0, 5)
            rows.append((ts[f], b[0], b[1], b[2], b[3], b[4], 0.5, tid))
    tr = np.array(rows, dtype=np.dtype([("t", "<u8"), ("x", "<f4"), ("y", "<f4"), ("w", "<f4"), ("h", "<f4"), ("class_id", "u1"),
                                        ("class_confidence", "<f4"), ("track_id", "<u4")]))
    return tr[np.argsort(tr["t"], kind="stable")], ts


@pytest.mark.parametrize("seed", range(6))
def test_product_pair_labels_equal_the_oracle_on_random_recordings(seed):
    tracks, ts = _random_recording(seed)
    pl = L.pair_labels(tracks, ts, SOURCE, W, H, SCALE, MIN_H, MIN_D)
    pairs, frames = R.recording_labels(tracks, ts, SOURCE, W, H, SCALE, MIN_H, MIN_D)
    assert np.array_equal(pl.pairs, pairs.reshape(-1, 2))
    assert len(pairs) > 3
    for p, (d0, d1) in enumerate(frames):
        a, b = pl.off[p], pl.off[p + 1]
        for box, d in ((pl.box0, d0), (pl.box1, d1)):
            assert same(box[a:b], np.stack([d[k] for k in "xywh"], 1).astype(np.float32))
        assert np.array_equal(pl.cls[a:b], d0["class_id"].astype(np.int64))


def test_bad_recordings_raise():
    tracks, ts = rec("rec_a")
    args = (SOURCE, W, H, SCALE, MIN_H, MIN_D)
    dup = tracks.copy()
    sel = np.flatnonzero(dup["t"] == ts[0])
    dup["track_id"][sel[1]] = dup["track_id"][sel[0]]
    dup["track_id"][np.flatnonzero(dup["t"] == ts[1])[1]] = dup["track_id"][sel[0]]
    with pytest.raises(ValueError, match="twice"):
        L.pair_labels(dup, ts, *args)
    back = ts.copy()
    back[1] = back[0]                                                          # t0 >= t1 for the pair (0, 1)
    moved = tracks.copy()
    moved["t"][moved["t"] == ts[1]] = ts[0]
    with pytest.raises(ValueError):
        L.pair_labels(moved[np.argsort(moved["t"], kind="stable")], back, *args)
    with pytest.raises(ValueError, match="sorted"):
        L.pair_labels(tracks[::-1], ts, *args)
    with pytest.raises(ValueError, match="fields"):
        L.pair_labels(np.zeros(3, dtype=[("t", "<u8"), ("x", "<f4")]), ts, *args)
    f64 = np.zeros(len(tracks), dtype=[(n, "<f8" if n in "xywh" else tracks.dtype[n]) for n in tracks.dtype.names])
    with pytest.raises(ValueError, match="float32"):
        L.pair_labels(f64, ts, *args)
    with pytest.raises(ValueError, match="class_id"):
        L.pair_labels(tracks, ts, SOURCE[:3], W, H, SCALE, MIN_H, MIN_D)
