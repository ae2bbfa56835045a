"""numpy restatement of the reference's DSEC label chain for the interframe evaluation (TEST INFRASTRUCTURE ONLY -- never
imported by the product path), written against structured track arrays as the reference uses them:

  src/dagr/data/dsec_utils.py       construct_pairs, rescale_tracks, crop_tracks, map_classes, filter_small_bboxes,
                                    filter_tracks (only_perfect_tracks=True), filter_by_only_perfect_tracks,
                                    is_invalid_track, compute_iou, compute_img_idx_to_track_idx, compute_class_mapping
  src/dagr/data/dsec_data.py        interpolate_tracks, DSEC.MAPPING, DSEC.preprocess_detections, the label half of
                                    DSEC.__getitem__ (tracks_to_array, the test-time transform, filter_small_bboxes)
  src/dagr/data/augment.py          Crop([0, 0], [1, 1]) on the boxes (_crop_bbox): clamp to [0, W-1] x [0, H-1]
  src/dagr/model/utils.py           convert_to_evaluation_format: x2 = x + w, y2 = y + h

`get_tracks(index, mask=...)` of dsec_det is not part of the reference tree: it is restated as the rows with
t == image_ts[index] that the track mask keeps, the slicing filter_by_only_perfect_tracks itself relies on.

interpolate_tracks has two numerical rules (RULES):
  'numpy1'  NumPy 1.x value-based casting, what the reference ran under (Python 3.8): r = (t - t0) / (t1 - t0) in float64,
            r and 1 - r each rounded to float32, x0 * (1 - r) + x1 * r computed in float32;
  'nep50'   NumPy 2 (NEP 50): the same expression in float64, rounded once to the float32 field.
dagr_b200's interframe_targets kernel follows 'numpy1'.  Pinned by tests/golden/interframe_labels_golden.npz, made from
the reference's unmodified functions (tests/golden/make_interframe_labels_golden.py)."""
from __future__ import annotations

import numpy as np

MAPPING = dict(pedestrian="pedestrian", rider=None, car="car", bus="car", truck="car", bicycle=None, motorcycle=None, train=None)
CLASSES = ("car", "pedestrian")
RULES = ("numpy1", "nep50")


def compute_class_mapping(classes, all_classes, mapping):
    return np.array([classes.index(mapping[c]) if mapping[c] in classes else -1 for c in all_classes])


def map_classes(class_ids, old_to_new):
    new = old_to_new[class_ids]
    return new, new > -1


def rescale_tracks(tracks, scale):
    out = tracks.copy()
    for k in "xywh":
        out[k] /= scale
    return out


def crop_tracks(tracks, width, height):
    out = tracks.copy()
    x1, y1 = out["x"], out["y"]
    x2, y2 = x1 + out["w"], y1 + out["h"]
    x1, x2 = np.clip(x1, 0, width - 1), np.clip(x2, 0, width - 1)
    y1, y2 = np.clip(y1, 0, height - 1), np.clip(y2, 0, height - 1)
    out["x"], out["y"], out["w"], out["h"] = x1, y1, x2 - x1, y2 - y1
    return out


def filter_small_bboxes(w, h, bbox_height, bbox_diag):
    diag = np.sqrt(h ** 2 + w ** 2)
    return (diag > bbox_diag) & (w > bbox_height) & (h > bbox_height)


def construct_pairs(indices):
    """(i, i + 1) for every i with both i and i + 1 in `indices` -> int [P, 2]"""
    s = np.sort(np.asarray(indices))
    keep = s[1:] == s[:-1] + 1
    return np.stack([s[:-1][keep], s[1:][keep]], axis=1)


def compute_iou(a, b):
    x1, x2, y1, y2 = a["x"], a["x"] + a["w"], a["y"], a["y"] + a["h"]
    gx1, gx2, gy1, gy2 = b["x"], b["x"] + b["w"], b["y"], b["y"] + b["h"]
    ix1, iy1 = np.maximum(x1, gx1), np.maximum(y1, gy1)
    ix2, iy2 = np.minimum(x2, gx2), np.minimum(y2, gy2)
    inter = np.zeros_like(x1)
    m = (iy2 > iy1) & (ix2 > ix1)
    inter[m] = (ix2[m] - ix1[m]) * (iy2[m] - iy1[m])
    union = (x2 - x1) * (y2 - y1) + (gx2 - gx1) * (gy2 - gy1) - inter + 1e-9
    return inter / union


def is_invalid_track(frames):
    a, b = (f[f["track_id"].argsort()] for f in frames)
    if len(a) != len(b) or not (a["track_id"] == b["track_id"]).all():
        return True
    return bool(np.min(compute_iou(a, b)) < 0.10)


def filter_tracks(tracks, image_ts, width, height, class_remapping, min_bbox_height, min_bbox_diag, scale):
    """one recording, only_perfect_tracks=True -> (pairs int [P, 2], track mask bool [n])"""
    rs = crop_tracks(rescale_tracks(tracks, scale), width, height)
    _, class_mask = map_classes(rs["class_id"], class_remapping)
    mask = filter_small_bboxes(rs["w"], rs["h"], min_bbox_height, min_bbox_diag) & class_mask
    valid = np.unique(np.nonzero(np.isin(image_ts, rs[mask]["t"]))[0])
    pairs = construct_pairs(valid)
    # compute_img_idx_to_track_idx: [start, end) of each distinct t (tracks sorted by t), for the pairs' two timestamps;
    # filter_by_only_perfect_tracks then compares rows [start(t0), start(t1)) with rows [end(t0), end(t1))
    ut, counts = np.unique(tracks["t"], return_counts=True)
    bounds = np.concatenate([[0], counts]).cumsum()
    keep = np.ones(len(pairs), bool)
    for i, (i0, i1) in enumerate(pairs):
        j0, j1 = np.searchsorted(ut, image_ts[i0]), np.searchsorted(ut, image_ts[i1])
        sl = [slice(bounds[j0], bounds[j1]), slice(bounds[j0 + 1], bounds[j1 + 1])]
        keep[i] = not is_invalid_track([rs[s][mask[s]] for s in sl])
    return pairs[keep], mask


def get_tracks(tracks, image_ts, index, mask):
    return tracks[(tracks["t"] == image_ts[index]) & mask]


def preprocess_detections(det, scale, width, height, class_remapping):
    det = crop_tracks(rescale_tracks(det, scale), width, height)
    det["class_id"], _ = map_classes(det["class_id"], class_remapping)
    return det


def sorted_by_track(det):
    return det[det["track_id"].argsort(kind="stable")]


def interpolate_tracks(d0, d1, t, rule="numpy1"):
    """d0, d1 sorted by track_id, t0 = d0['t'][0] < t1 = d1['t'][0]; class ids and track ids from d0."""
    assert len(d0) == len(d1)
    if len(d0) == 0:
        return d1.copy()
    t0, t1 = int(d0["t"][0]), int(d1["t"][0])
    assert t0 < t1
    r = (int(t) - t0) / (t1 - t0)
    out = d0.copy()
    for k in "xywh":
        if rule == "numpy1":
            out[k] = d0[k] * np.float32(1 - r) + d1[k] * np.float32(r)
        elif rule == "nep50":
            out[k] = (d0[k].astype(np.float64) * (1 - r) + d1[k].astype(np.float64) * r).astype(np.float32)
        else:
            raise ValueError(rule)
    return out


def test_time_targets(det, width, height, min_bbox_height, min_bbox_diag):
    """tracks_to_array -> Crop([0, 0], [1, 1]) -> filter_small_bboxes -> convert_to_evaluation_format, in float32:
    -> (boxes f32 [n, 4] xyxy, labels i64 [n])"""
    x, y = det["x"].astype(np.float32), det["y"].astype(np.float32)
    x2, y2 = x + det["w"].astype(np.float32), y + det["h"].astype(np.float32)
    x, x2 = np.clip(x, 0, width - 1), np.clip(x2, 0, width - 1)
    y, y2 = np.clip(y, 0, height - 1), np.clip(y2, 0, height - 1)
    w, h = x2 - x, y2 - y
    keep = filter_small_bboxes(w, h, min_bbox_height, min_bbox_diag)
    boxes = np.stack([x, y, x + w, y + h], axis=1)[keep].astype(np.float32)
    return boxes.reshape(-1, 4), det["class_id"][keep].astype(np.int64)


def recording_labels(tracks, image_ts, source_classes, width, height, scale=2, min_bbox_height=0, min_bbox_diag=0):
    """-> (pairs int [P, 2], [(d0, d1)] the pairs' preprocessed frame labels, each sorted by track_id)"""
    remap = compute_class_mapping(CLASSES, list(source_classes), MAPPING)
    image_ts = np.asarray(image_ts)
    pairs, mask = filter_tracks(tracks, image_ts, width, height, remap, min_bbox_height, min_bbox_diag, scale)
    frames = [tuple(sorted_by_track(preprocess_detections(get_tracks(tracks, image_ts, i, mask), scale, width, height, remap))
                    for i in (i0, i1)) for i0, i1 in pairs]
    return pairs, frames


def window_targets(d0, d1, t, width, height, min_bbox_height, min_bbox_diag, rule="numpy1"):
    """the ground truth of the window [t0, t) of one pair, as the evaluation sees it"""
    return test_time_targets(interpolate_tracks(d0, d1, t, rule), width, height, min_bbox_height, min_bbox_diag)


def flat_targets(box0, box1, cls, pair_off, pair_t, win_pair, win_t, win_group, K, width, height, min_bbox_height, min_bbox_diag):
    """window_targets under 'numpy1' for many windows at once, in the flat layout of dagr_interframe_targets:
    label tables box0 / box1 f32 [n, 4] xywh, cls [n], pair p owning rows [pair_off[p], pair_off[p+1]) with
    pair_t[p] = (t0, t1); window w = (win_pair[w], win_t[w], win_group[w]).  -> (gt_box f32 [m, 4] xyxy,
    gt_label i64 [m] = group * K + class, gt_off i64 [Q + 1])"""
    pair_off, pair_t = np.asarray(pair_off, np.int64), np.asarray(pair_t, np.int64).reshape(-1, 2)
    win_pair, win_t = np.asarray(win_pair, np.int64), np.asarray(win_t, np.int64)
    n = pair_off[win_pair + 1] - pair_off[win_pair]
    w = np.repeat(np.arange(len(win_pair)), n)
    row = pair_off[win_pair][w] + (np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n))
    p = win_pair[w]
    r = (win_t[w] - pair_t[p, 0]).astype(np.float64) / (pair_t[p, 1] - pair_t[p, 0]).astype(np.float64)
    fr, fq = r.astype(np.float32), (1.0 - r).astype(np.float32)
    v = box0[row] * fq[:, None] + box1[row] * fr[:, None]                  # float32 throughout
    det = np.zeros(len(row), dtype=[("x", "<f4"), ("y", "<f4"), ("w", "<f4"), ("h", "<f4"), ("class_id", "<i8")])
    det["x"], det["y"], det["w"], det["h"] = v[:, 0], v[:, 1], v[:, 2], v[:, 3]
    det["class_id"] = np.asarray(win_group, np.int64)[w] * K + np.asarray(cls, np.int64)[row]
    x, y = det["x"], det["y"]
    x2, y2 = np.clip(x + det["w"], 0, width - 1), np.clip(y + det["h"], 0, height - 1)
    x, y = np.clip(x, 0, width - 1), np.clip(y, 0, height - 1)
    ww, hh = x2 - x, y2 - y
    keep = filter_small_bboxes(ww, hh, min_bbox_height, min_bbox_diag)
    boxes = np.stack([x, y, x + ww, y + hh], axis=1)[keep].astype(np.float32).reshape(-1, 4)
    off = np.concatenate([[0], np.cumsum(np.bincount(w[keep], minlength=len(win_pair)))]).astype(np.int64)
    return boxes, det["class_id"][keep], off
