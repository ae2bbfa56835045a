#!/usr/bin/env python
"""Generate tests/golden/interframe_labels_golden.npz from the REFERENCE's own, unmodified label chain (build container
only; no test imports this file):

  src/dagr/data/dsec_utils.py   filter_tracks (only_perfect_tracks=True) with everything it calls, compute_class_mapping
  src/dagr/data/dsec_data.py    interpolate_tracks, DSEC.MAPPING, DSEC.preprocess_detections, tracks_to_array,
                                filter_small_bboxes on the transformed boxes (DSEC.__getitem__)
  src/dagr/data/augment.py      Crop([0, 0], [1, 1]) initialised at the dataset's height and width (transform_testing)

The modules are imported as written; h5py, dsec_det, torch_geometric, numba and cv2 are replaced by stand-ins that hold
only the names the imports need (none of their code runs here).  dsec_det's get_tracks(index, mask=...) is not in the
reference tree and is restated as the rows with t == image_ts[index] that the track mask keeps.

interpolate_tracks runs twice per window: as is, under the installed NumPy 2 (NEP 50: float64 arithmetic, one rounding),
and fed label arrays whose 't' field holds Python ints (and a Python int t), so that r is a Python float and the
arithmetic is float32 with r and 1 - r rounded first -- the promotion NumPy 1 gave the reference.  The shim changes the
inputs, not the function."""
import sys
import types
from pathlib import Path

import numpy as np
import torch

REF_SRC = "/root/reference/src"
OUT = Path(__file__).resolve().parent / "interframe_labels_golden.npz"

# ---- stand-ins for the third-party imports ---------------------------------------------------------------------------


def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__path__ = []
    m.__dict__.update(attrs)
    sys.modules[name] = m
    if "." in name:
        parent, child = name.rsplit(".", 1)
        setattr(sys.modules[parent], child, m)
    return m


class Data:
    def __init__(self, **kw):
        self.__dict__.update(kw)


class BaseTransform:
    pass


class Compose:
    def __init__(self, transforms):
        self.transforms = transforms

    def __call__(self, data):
        for t in self.transforms:
            data = t(data)
        return data


def _identity_decorator(*a, **k):
    if len(a) == 1 and callable(a[0]) and not k:
        return a[0]
    return lambda f: f


_mod("h5py", File=None)
_mod("cv2", resize=None, imshow=None, waitKey=None, INTER_CUBIC=2, INTER_NEAREST=0)
_mod("numba", njit=_identity_decorator, jit=_identity_decorator)
_mod("torch_geometric")
_mod("torch_geometric.data", Data=Data, Dataset=object)
_mod("torch_geometric.transforms", BaseTransform=BaseTransform, Compose=Compose)
_mod("dsec_det")
_mod("dsec_det.dataset", DSECDet=None)
_mod("dsec_det.io", yaml_file_to_dict=None)
_mod("dsec_det.directory", BaseDirectory=object)
_mod("torchvision")
sys.path.insert(0, REF_SRC)

from dagr.data import dsec_utils as U          # noqa: E402
from dagr.data import dsec_data as D           # noqa: E402
from dagr.data import augment as A             # noqa: E402

# ---- the recording ---------------------------------------------------------------------------------------------------
SOURCE = ("pedestrian", "rider", "car", "bus", "truck", "bicycle", "motorcycle", "train")
W, H, SCALE, MIN_H, MIN_D = 320, 215, 2, 10, 15
TRACK_DTYPE = np.dtype([("t", "<u8"), ("x", "<f4"), ("y", "<f4"), ("w", "<f4"), ("h", "<f4"), ("class_id", "u1"),
                        ("class_confidence", "<f4"), ("track_id", "<u4")])
OFFSETS = [int(v) for v in np.linspace(0, 50_000, 11)] + [1, 33_333, 49_999]


def _rescaled_iou(a, b):
    """compute_iou of two raw boxes (x, y, w, h) after the dataset's rescale and crop"""
    tr = np.zeros(2, TRACK_DTYPE)
    for i, (x, y, w, h) in enumerate((a, b)):
        tr[i]["x"], tr[i]["y"], tr[i]["w"], tr[i]["h"] = x, y, w, h
    tr = U.crop_tracks(U.rescale_tracks(tr, SCALE), W, H)
    return U.compute_iou(tr[:1], tr[1:])[0]


def _iou_edge():
    """the raw x of a second box where compute_iou crosses 0.10: (x just kept, next float32 just dropped)"""
    a = (200.0, 200.0, 60.0, 60.0)
    lo, hi = np.float32(200.0), np.float32(300.0)                  # iou(lo) >= 0.1 > iou(hi)
    while np.nextafter(lo, hi) != hi:
        mid = np.float32((float(lo) + float(hi)) / 2)
        if mid in (lo, hi):
            mid = np.nextafter(lo, hi)
        lo, hi = (mid, hi) if _rescaled_iou(a, (mid, 200.0, 60.0, 60.0)) >= 0.10 else (lo, mid)
    assert _rescaled_iou(a, (lo, 200.0, 60.0, 60.0)) >= 0.10 > _rescaled_iou(a, (hi, 200.0, 60.0, 60.0))
    return a, lo, hi


def _diag_edge():
    """raw w = h where the rescaled box's float32 diagonal crosses MIN_D: (largest w dropped, smallest w kept)"""
    w = np.float32(MIN_D / np.sqrt(2) * SCALE)
    diag = lambda v: np.sqrt((v / np.float32(SCALE)) ** 2 + (v / np.float32(SCALE)) ** 2)
    while diag(w) > MIN_D:
        w = np.nextafter(w, np.float32(0))
    while not diag(np.nextafter(w, np.float32(100))) > MIN_D:
        w = np.nextafter(w, np.float32(100))
    return w, np.nextafter(w, np.float32(100))


def recording(seed, t_start, intervals):
    rng = np.random.default_rng(seed)
    ts = np.concatenate([[t_start], t_start + np.cumsum(intervals)]).astype(np.int64)
    rows = []

    def add(f, tid, cls, x, y, w, h):
        rows.append((int(ts[f]), x, y, w, h, cls, 0.9, tid))

    # frames 0..2: three moving tracks and a rider (mapped to None), rows out of track order; frame 3 has no labels
    for f in range(3):
        for tid, cls, x, y in ((9, 2, 100.0, 120.0), (2, 0, 400.0, 200.0), (5, 4, 250.0, 300.0)):
            jx, jy, jw, jh = rng.normal(0, 6, 4)
            add(f, tid, cls, x + 13.7 * f + jx, y - 7.3 * f + jy, 61.3 + jw, 47.9 + jh)
        add(f, 40, 1, 300.0 + f, 100.0, 50.0, 90.0)
    # frames 4, 5: the track ids differ
    add(4, 1, 2, 100.0, 100.0, 80.0, 60.0)
    add(5, 3, 2, 104.0, 100.0, 80.0, 60.0)
    # frames 6, 7: IoU just under 0.10; frames 8, 9: just over
    a, keep_x, drop_x = _iou_edge()
    add(6, 7, 2, *a)
    add(7, 7, 2, float(drop_x), 200.0, 60.0, 60.0)
    add(8, 7, 2, *a)
    add(9, 7, 2, float(keep_x), 200.0, 60.0, 60.0)
    # frames 10, 11: boxes crossing every border, one beyond the right edge (clamped to zero width), classes mapped to
    # None, and size filters one ulp either side of MIN_H and MIN_D (at x = y = 0, where x + w is exact)
    lo_d, hi_d = _diag_edge()
    h_in, h_out = np.nextafter(np.float32(2 * MIN_H), np.float32(100)), np.float32(2 * MIN_H)
    for f in (10, 11):
        s = f - 10
        add(f, 11, 2, -30.0 + 9 * s, 50.0, 120.0, 70.0)                   # left
        add(f, 12, 0, 560.0 - 7 * s, 60.0, 110.0, 120.0)                  # right
        add(f, 13, 3, 200.0, -40.0 + 5 * s, 90.0, 100.0)                  # top
        add(f, 14, 4, 300.0, 380.0 + 4 * s, 100.0, 80.0)                  # bottom (cropped height 430)
        add(f, 15, 2, -50.0, -50.0 - s, 700.0, 600.0)                     # every border at once
        add(f, 16, 2, 700.0, 100.0, 40.0, 40.0)                           # beyond the right edge: zero width
        add(f, 17, 5, 100.0, 300.0, 60.0, 60.0)                           # bicycle -> None
        add(f, 18, 2, 0.0, 250.0, float(h_in), 80.0)                      # width one ulp over MIN_H: kept
        add(f, 19, 2, 0.0, 330.0, float(h_out), 80.0)                     # width exactly MIN_H: dropped
        add(f, 20, 2, 0.0, 0.0, float(hi_d), float(hi_d))                 # diagonal just over MIN_D (w, h > MIN_H)
        add(f, 21, 2, 0.0, 0.0, float(lo_d), float(lo_d))                 # diagonal not over MIN_D
        add(f, 22, 0, 150.0 + 8 * s, 150.0, 60.0 - 36 * s, 70.0 - 26 * s)    # shrinks: extrapolated past the filter
    # frames 12..14: two tracks, then one dies and another is born in frame 14
    for f, tids in ((12, (30, 31)), (13, (30, 31)), (14, (30, 32))):
        for tid in tids:
            add(f, tid, 2, 50.0 + 40 * tid - 1100 + 11 * f, 150.0 + 3 * f, 70.0, 50.0)
    tracks = np.array(rows, dtype=TRACK_DTYPE)
    tracks = tracks[np.argsort(tracks["t"], kind="stable")]
    return tracks, ts


RECORDINGS = {
    "rec_a": recording(1, 51_000_000_123, [50_000] * 8 + [49_999, 50_000, 50_001, 50_000, 50_000, 50_000]),
    "rec_b": recording(2, 7_000_000, [50_000, 40_000, 50_000, 50_000, 50_000, 50_000, 50_000, 50_000, 50_000, 50_000,
                                      25_000, 50_000, 50_000, 50_000]),
}


class _Dir:
    def __init__(self, name, tracks, ts):
        self.name = name
        self.tracks = types.SimpleNamespace(tracks=tracks)
        self.images = types.SimpleNamespace(timestamps=ts)


def _with_int_t(det):
    """the same rows with an object 't' field (Python ints): NumPy 1's promotion of r under NEP 50"""
    dt = np.dtype([(n, object if n == "t" else det.dtype[n]) for n in det.dtype.names])
    out = np.zeros(len(det), dt)
    for n in det.dtype.names:
        out[n] = [int(v) for v in det[n]] if n == "t" else det[n]
    return out


def targets(det):
    data = Data(bbox=torch.from_numpy(D.tracks_to_array(det)), x=torch.zeros((0, 1)), pos=torch.zeros((0, 2), dtype=torch.int16))
    transform = Compose([A.Crop([0, 0], [1, 1])])
    A.init_transforms(transform.transforms, H, W)
    data = transform(data)
    keep = D.filter_small_bboxes(data.bbox[:, 2], data.bbox[:, 3], MIN_H, MIN_D)
    bbox = data.bbox[keep].clone()
    bbox[:, 2:4] += bbox[:, :2]                                             # convert_to_evaluation_format
    return bbox[:, :4].numpy().astype(np.float32).reshape(-1, 4), bbox[:, 4].long().numpy()


def main():
    remap = U.compute_class_mapping(("car", "pedestrian"), SOURCE, D.DSEC.MAPPING)
    dataset = types.SimpleNamespace(subsequence_directories=[], directories={})
    for name, (tracks, ts) in RECORDINGS.items():
        d = _Dir(name, tracks, ts)
        dataset.subsequence_directories.append(d)
        dataset.directories[name] = d
    pairs_all, masks = U.filter_tracks(dataset=dataset, image_width=W, image_height=H, class_remapping=remap, min_bbox_height=MIN_H,
                                       min_bbox_diag=MIN_D, only_perfect_tracks=True, scale=SCALE)
    fake = types.SimpleNamespace(scale=SCALE, width=W, height=H, class_remapping=remap)
    out = dict(source=np.array(SOURCE), dims=np.array([W, H, SCALE, MIN_H, MIN_D]), offsets=np.array(OFFSETS))
    for name, (tracks, ts) in RECORDINGS.items():
        pairs, mask = pairs_all[name], masks[name]
        out[f"{name}_tracks"], out[f"{name}_image_ts"], out[f"{name}_pairs"], out[f"{name}_mask"] = tracks, ts, pairs, mask
        frames = []
        for i0, i1 in pairs:
            f = [D.DSEC.preprocess_detections(fake, tracks[(tracks["t"] == ts[i]) & mask]) for i in (i0, i1)]
            frames.append([x[x["track_id"].argsort()] for x in f])
        n = [len(f0) for f0, _ in frames]
        out[f"{name}_off"] = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
        for j in (0, 1):
            rows = np.concatenate([f[j] for f in frames]) if frames else np.zeros(0, TRACK_DTYPE)
            out[f"{name}_box{j}"] = np.stack([rows[k] for k in "xywh"], axis=1).astype(np.float32).reshape(-1, 4)
            out[f"{name}_cls{j}"] = rows["class_id"].astype(np.int64)
            out[f"{name}_tid{j}"] = rows["track_id"].astype(np.int64)
        for rule in ("nep50", "numpy1"):
            boxes, labels, off = [], [], [0]
            for n_us in OFFSETS:                                                # offset-major, then pair
                for (i0, _), (f0, f1) in zip(pairs, frames):
                    t = int(ts[i0]) + n_us
                    if rule == "nep50":
                        det = D.interpolate_tracks(f0, f1, np.int64(ts[i0]) + np.int64(n_us))
                    else:
                        det = D.interpolate_tracks(_with_int_t(f0), _with_int_t(f1), t)
                    b, lab = targets(det)
                    boxes.append(b)
                    labels.append(lab)
                    off.append(off[-1] + len(b))
            out[f"{name}_{rule}_box"] = np.concatenate(boxes).reshape(-1, 4)
            out[f"{name}_{rule}_label"] = np.concatenate(labels).astype(np.int64)
            out[f"{name}_{rule}_off"] = np.array(off, dtype=np.int64)
    np.savez_compressed(OUT, **out)
    for name in RECORDINGS:
        print(name, "pairs", out[f"{name}_pairs"].tolist(), "rows", len(out[f"{name}_box0"]),
              "targets", len(out[f"{name}_numpy1_box"]),
              "rule bits differ", int((out[f"{name}_numpy1_box"].view(np.int32) != out[f"{name}_nep50_box"].view(np.int32)).sum())
              if len(out[f"{name}_numpy1_box"]) == len(out[f"{name}_nep50_box"]) else "in count")


if __name__ == "__main__":
    main()
