"""The reference's DSEC label chain on the host, as pure functions over arrays: which frame pairs a recording contributes to
the interframe evaluation, and each pair's labels after DSEC.preprocess_detections.

  src/dagr/data/dsec_utils.py   compute_class_mapping, map_classes, rescale_tracks, crop_tracks, filter_small_bboxes,
                                filter_tracks with only_perfect_tracks=True (construct_pairs, compute_img_idx_to_track_idx,
                                filter_by_only_perfect_tracks, is_invalid_track, compute_iou)
  src/dagr/data/dsec_data.py    DSEC.MAPPING, DSEC.preprocess_detections (rescale, crop, class mapping)

This is once-per-recording work; the per-window half of the chain (interpolate_tracks, the test-time Crop, the size filter,
the evaluation format) runs on the device in dagr_interframe_targets (dagr_b200.interframe).

A recording is its `tracks` structured array (fields t, x, y, w, h, class_id, track_id; x, y, w, h float32; t sorted, as
DSEC stores it) and its image timestamps.  The labels of frame i are the rows with t == image_ts[i] that the track mask of
filter_tracks keeps: dsec_det's get_tracks(i, mask=...) restated, and the slicing filter_by_only_perfect_tracks relies on.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

MAPPING = dict(pedestrian="pedestrian", rider=None, car="car", bus="car", truck="car", bicycle=None, motorcycle=None, train=None)
CLASSES = ("car", "pedestrian")
FIELDS = ("t", "x", "y", "w", "h", "class_id", "track_id")


def compute_class_mapping(classes, all_classes, mapping=MAPPING) -> np.ndarray:
    """source class index -> index in `classes`, or -1 where the mapping drops the class"""
    return np.array([classes.index(mapping[c]) if mapping[c] in classes else -1 for c in all_classes], dtype=np.int64)


def map_classes(class_ids, old_to_new):
    new = np.asarray(old_to_new)[np.asarray(class_ids)]
    return new, new > -1


def rescale_tracks(x, y, w, h, scale):
    return tuple((v / np.float32(scale)).astype(np.float32) for v in (x, y, w, h))


def crop_tracks(x, y, w, h, width, height):
    """clip both corners to [0, width-1] x [0, height-1] in float32 -> (x, y, w, h)"""
    x2, y2 = x + w, y + h
    x, x2 = np.clip(x, np.float32(0), np.float32(width - 1)), np.clip(x2, np.float32(0), np.float32(width - 1))
    y, y2 = np.clip(y, np.float32(0), np.float32(height - 1)), np.clip(y2, np.float32(0), np.float32(height - 1))
    return x, y, x2 - x, y2 - y


def filter_small_bboxes(w, h, bbox_height, bbox_diag):
    """float32 sqrt(h*h + w*w) > bbox_diag and w, h > bbox_height (strict)"""
    w, h = np.asarray(w, np.float32), np.asarray(h, np.float32)
    return (np.sqrt(h * h + w * w) > np.float32(bbox_diag)) & (w > np.float32(bbox_height)) & (h > np.float32(bbox_height))


def compute_iou(b0, b1):
    """float32 IoU of paired xywh rows [n, 4], with the reference's + 1e-9 in the union"""
    x1, y1, x2, y2 = b0[:, 0], b0[:, 1], b0[:, 0] + b0[:, 2], b0[:, 1] + b0[:, 3]
    gx1, gy1, gx2, gy2 = b1[:, 0], b1[:, 1], b1[:, 0] + b1[:, 2], b1[:, 1] + b1[:, 3]
    ix1, iy1, ix2, iy2 = np.maximum(x1, gx1), np.maximum(y1, gy1), np.minimum(x2, gx2), np.minimum(y2, gy2)
    inter = np.where((iy2 > iy1) & (ix2 > ix1), (ix2 - ix1) * (iy2 - iy1), np.float32(0))
    union = (x2 - x1) * (y2 - y1) + (gx2 - gx1) * (gy2 - gy1) - inter + np.float32(1e-9)
    return inter / union


@dataclass
class PairLabels:
    """the kept (i0, i1) pairs of one recording and the preprocessed labels of both frames, paired row by row.
    Pair p owns rows [off[p], off[p+1]) of box0 / box1 (xywh float32, frames i0 and i1), cls (class index from frame
    i0) and track_id, sorted by track_id; t[p] = (image_ts[i0], image_ts[i1])."""
    pairs: np.ndarray          # int64 [P, 2]
    t: np.ndarray              # int64 [P, 2]
    off: np.ndarray            # int64 [P + 1]
    box0: np.ndarray           # float32 [n, 4]
    box1: np.ndarray           # float32 [n, 4]
    cls: np.ndarray            # int64 [n]
    track_id: np.ndarray       # int64 [n]

    def __len__(self):
        return len(self.pairs)


def _check(tracks, image_ts):
    names = tracks.dtype.names or ()
    missing = [f for f in FIELDS if f not in names]
    if missing:
        raise ValueError(f"tracks lacks the fields {missing} (expected {FIELDS})")
    for k in "xywh":
        if tracks.dtype[k] != np.float32:
            raise ValueError(f"tracks[{k!r}] is {tracks.dtype[k]}: expected float32")
    for k in ("t", "class_id", "track_id"):
        if tracks.dtype[k].kind not in "iu":
            raise ValueError(f"tracks[{k!r}] is {tracks.dtype[k]}: expected integers")
    t = tracks["t"].astype(np.int64)
    if len(t) > 1 and (np.diff(t) < 0).any():
        raise ValueError("tracks must be sorted by t")
    ts = np.asarray(image_ts)
    if ts.dtype.kind not in "iu":
        raise ValueError(f"image timestamps of dtype {ts.dtype}: expected integer microseconds")
    return t, ts.astype(np.int64).reshape(-1)


def pair_labels(tracks, image_ts, source_classes, width: int, height: int, scale: int = 2, min_bbox_height=0,
                min_bbox_diag=0) -> PairLabels:
    """filter_tracks(only_perfect_tracks=True) and, per kept pair, preprocess_detections of both frames' labels.
    width, height: the model's (cropped) resolution; scale: sensor pixels per model pixel.  Raises ValueError on a
    malformed track array, on a kept pair whose frames are not strictly increasing in time, and on a track_id that
    appears twice in one frame of a kept pair (the reference's sort would leave that order undefined)."""
    t, image_ts = _check(tracks, image_ts)
    remap = compute_class_mapping(CLASSES, list(source_classes))
    cid = tracks["class_id"].astype(np.int64)
    if len(cid) and (cid.min() < 0 or cid.max() >= len(remap)):
        raise ValueError(f"class_id outside [0, {len(remap)}) for {len(remap)} source classes")
    x, y, w, h = crop_tracks(*rescale_tracks(tracks["x"], tracks["y"], tracks["w"], tracks["h"], scale), width, height)
    cls, class_mask = map_classes(cid, remap)
    mask = filter_small_bboxes(w, h, min_bbox_height, min_bbox_diag) & class_mask
    valid = np.unique(np.nonzero(np.isin(image_ts, t[mask]))[0])
    first = valid[:-1][valid[1:] == valid[:-1] + 1]                          # construct_pairs: consecutive image indices
    pairs = np.stack([first, first + 1], axis=1).astype(np.int64)
    box = np.stack([x, y, w, h], axis=1)
    tid = tracks["track_id"].astype(np.int64)

    def frame(a, b):                                    # kept rows of [a, b), sorted by track_id
        r = np.arange(a, b)[mask[a:b]]
        return r[np.argsort(tid[r], kind="stable")]

    keep, rows0, rows1 = [], [], []
    for i0, i1 in pairs:
        t0, t1 = image_ts[i0], image_ts[i1]
        s0, e0 = np.searchsorted(t, t0, "left"), np.searchsorted(t, t0, "right")
        s1, e1 = np.searchsorted(t, t1, "left"), np.searchsorted(t, t1, "right")
        if t0 >= t1:
            raise ValueError(f"pair ({i0}, {i1}): image timestamps {t0} >= {t1}")
        # filter_by_only_perfect_tracks compares rows [start(t0), start(t1)) with [end(t0), end(t1))
        a, b = frame(s0, s1), frame(e0, e1)
        if len(a) != len(b) or not np.array_equal(tid[a], tid[b]):
            continue
        if (np.diff(tid[a]) == 0).any():
            raise ValueError(f"pair ({i0}, {i1}): a track_id appears twice in one frame")
        if compute_iou(box[a], box[b]).min() < 0.10:
            continue
        f0, f1 = frame(s0, e0), frame(s1, e1)                                  # get_tracks of both frames
        if len(f0) != len(f1):
            raise ValueError(f"pair ({i0}, {i1}): {len(f0)} and {len(f1)} labels (track rows between the two frames)")
        keep.append((i0, i1))
        rows0.append(f0)
        rows1.append(f1)
    P = len(keep)
    n = np.array([len(r) for r in rows0], dtype=np.int64)
    r0 = np.concatenate(rows0) if P else np.zeros(0, np.int64)
    r1 = np.concatenate(rows1) if P else np.zeros(0, np.int64)
    pr = np.array(keep, dtype=np.int64).reshape(P, 2)
    return PairLabels(pr, image_ts[pr].reshape(P, 2), np.concatenate([[0], np.cumsum(n)]).astype(np.int64),
                      box[r0].astype(np.float32).reshape(-1, 4), box[r1].astype(np.float32).reshape(-1, 4), cls[r0], tid[r0])
