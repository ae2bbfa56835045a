#!/usr/bin/env python
"""Generate tests/golden/ingest_window_golden.npz from the REFERENCE's own event preprocessing (build container only):

    DAGR_REFERENCE=/path/to/uzh-rpg/dagr python tests/golden/make_ingest_window_golden.py

One DSEC sample's events go through the reference's unmodified code: `DSEC.preprocess_events` (dsec_data.py:141-147: crop
y < height, t = time_window + t - t[-1], p -> 2p - 1), called unbound on a namespace carrying height and time_window;
`dagr.data.utils.to_data` (x, y -> int16, t -> int32); `dagr.utils.buffers.format_data` (cat to int32, true division by
[W, H, T] in fp32); `dagr.model.layers.ev_tgn.denormalize_pos` ((pos * [W, H, T] + 1e-3).int()).  The one restated step is
the window cut `t < t_cut` of DSEC.__getitem__ (dsec_data.py:177-179), an inline expression there.  width, height and
time_window are set on the Data as the one-element tensors a collated batch carries.

Window cases c0..c10 (p stored in {0, 1} as u1; keys c{i}_in_{x,y,t,p}, c{i}_dims = [W, H, T], c{i}_t_cut, and the
reference's c{i}_pos i32[M, 3] and c{i}_feat f32[M]):
  c0   a random sorted window, 640 x 430 cropped from 480 rows
  c1   t == t_cut (cut) next to t_cut - 1 (kept)
  c2   y == H (cropped) next to H - 1 (kept)
  c3   the latest events cropped away: t[-1] is an earlier event's t
  c4   timestamp ties at the last event
  c5   a window cut to nothing
  c6   absolute timestamps above 2^32
  c7   x >= 32768, which wraps through int16
  c8   a window longer than 2^31 us: the relative t wraps through int32
  c9   an unsorted window: t[-1] is neither the largest nor the smallest kept t
  c10  an all-negative window

Denormalisation sweep: for every (W, H) in SWEEP_WH and T in SWEEP_T, a sorted window of T + 1 events with t = 0..T,
x = i % W, y = i % H, so that the relative t runs over every value of [0, T] and x, y over every column and row.  Only
the coordinates whose denormalised value differs from the input are stored, per axis: sweep_{x,y,t}{dim}_in / _out.  The
generator checks that every (W, H, T) combination gives the same exceptions per axis, so they are stored once per W, H or T.
"""
import os
import sys
import types
from pathlib import Path

import numpy as np
import torch

if not os.environ.get("DAGR_REFERENCE"):
    sys.exit("set DAGR_REFERENCE to an uzh-rpg/dagr checkout")
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
from tests.golden import ref_shim  # noqa: E402

ref_shim.REF_SRC = str(Path(os.environ["DAGR_REFERENCE"]) / "src")
ref_shim.install()
import dagr.data  # noqa: E402,F401  (the real package, before stubs are put under it)
for name in ("h5py", "hdf5plugin", "dsec_det", "dsec_det.dataset", "dsec_det.io", "dsec_det.directory", "pycocotools",
             "pycocotools.coco", "pycocotools.cocoeval", "detectron2", "detectron2.structures", "detectron2.evaluation",
             "detectron2.evaluation.fast_eval_api", "dagr.data.augment", "dagr.visualization", "dagr.visualization.bbox_viz",
             "dagr.visualization.event_viz"):
    ref_shim._mod(name)
sys.modules["torch_geometric.data"].Dataset = object
for mod, names in {"dsec_det.dataset": ["DSECDet"], "dsec_det.io": ["yaml_file_to_dict"], "dsec_det.directory": ["BaseDirectory"],
                   "dagr.data.augment": ["init_transforms"], "dagr.visualization.bbox_viz": ["draw_bbox_on_img"],
                   "dagr.visualization.event_viz": ["draw_events_on_image"], "pycocotools.coco": ["COCO"],
                   "pycocotools.cocoeval": ["COCOeval"], "detectron2.structures": ["Boxes", "BoxMode", "pairwise_iou"],
                   "detectron2.evaluation": ["COCOEvaluator"], "detectron2.evaluation.fast_eval_api": ["COCOeval_opt"]}.items():
    for n in names:
        setattr(sys.modules[mod], n, type(n, (), {}))                  # placeholders: never called here
from dagr.data.dsec_data import DSEC  # noqa: E402
from dagr.data.utils import to_data  # noqa: E402
from dagr.model.layers.ev_tgn import denormalize_pos  # noqa: E402
from dagr.utils.buffers import format_data  # noqa: E402

SWEEP_WH = [(640, 430), (320, 215), (240, 180), (1280, 720)]
SWEEP_T = [1_000_000, 50_000, 999_999]


def reference(ev, W, H, T, t_cut):
    """the reference's chain on one sample -> (pos_denorm i32[M, 3], polarity f32[M])."""
    ev = {k: v[ev["t"] < t_cut] for k, v in ev.items()}                     # dsec_data.py:177-179
    ev = DSEC.preprocess_events(types.SimpleNamespace(height=H, time_window=T), ev)
    data = to_data(**ev, width=W, height=H, time_window=T)
    data.width, data.height, data.time_window = torch.tensor([W]), torch.tensor([H]), torch.tensor([T])
    data = format_data(data)
    pos = denormalize_pos(data)
    assert pos.dtype == torch.int32 and data.x.dtype == torch.float32
    return pos.numpy(), data.x.reshape(-1).numpy()


rng = np.random.default_rng(19)
out = {}


def case(i, x, y, t, p, W, H, T, t_cut):
    ev = dict(x=np.asarray(x, np.uint16), y=np.asarray(y, np.uint16), t=np.asarray(t, np.int64), p=np.asarray(p, np.uint8))
    pos, feat = reference({k: v.copy() for k, v in ev.items()}, W, H, T, t_cut)
    for k, v in ev.items():
        out[f"c{i}_in_{k}"] = v
    out[f"c{i}_dims"] = np.array([W, H, T], np.int64)
    out[f"c{i}_t_cut"] = np.array(t_cut, np.int64)
    out[f"c{i}_pos"], out[f"c{i}_feat"] = pos, feat


def rand(n, W, Hs, t0, span, sort=True):
    t = t0 + rng.integers(0, span, n)
    return (rng.integers(0, W, n), rng.integers(0, Hs, n), np.sort(t) if sort else t, rng.integers(0, 2, n))


NO_CUT = 1 << 62
W, H, T = 640, 430, 1_000_000
x, y, t, p = rand(5000, W, 480, 7_000_000, 60_000)
case(0, x, y, t, p, W, H, T, 7_050_000)
x, y, t, p = rand(300, W, H, 7_000_000, 50_000)
t[-3:] = [7_049_999, 7_050_000, 7_050_000]
case(1, x, y, np.sort(t), p, W, H, T, 7_050_000)
x, y, t, p = rand(300, W, H, 7_000_000, 50_000)
y[-4:] = [H - 1, H, H - 1, H]
case(2, x, y, t, p, W, H, T, NO_CUT)
x, y, t, p = rand(400, W, H, 7_000_000, 50_000)
y[-25:] = rng.integers(H, 480, 25)
case(3, x, y, t, p, W, H, T, NO_CUT)
x, y, t, p = rand(400, W, H, 7_000_000, 50_000)
t[-6:] = t[-6]
case(4, x, y, t, p, W, H, T, NO_CUT)
x, y, t, p = rand(200, W, H, 7_000_000, 50_000)
case(5, x, y, t, p, W, H, T, 7_000_000)
x, y, t, p = rand(2000, W, H, (1 << 32) + 123_456_789, 900_000)
case(6, x, y, t, p, W, H, T, NO_CUT)
x, y, t, p = rand(2000, 65536, H, 7_000_000, 50_000)
x[:4] = [32767, 32768, 65535, 40000]
case(7, x, y, t, p, W, H, T, NO_CUT)
x, y, t, p = rand(3000, W, H, 5_000_000_000, 5_000_000_000)
t[0] = 5_000_000_000                                                   # the window spans more than 2^32 us
case(8, x, y, t, p, W, H, T, NO_CUT)
x, y, t, p = rand(3000, W, 480, 7_000_000, 60_000, sort=False)
t[-1] = 7_030_000
y[-1] = 5
case(9, x, y, t, p, W, H, T, 7_050_000)
x, y, t, p = rand(500, W, 480, -40_000, 39_000)
y[-1] = 470                                                            # the last kept event is not the last event
case(10, x, y, t, p, W, H, T, NO_CUT)

# the sweep
exc = {}
dims = []
for Wd, Hd in SWEEP_WH:
    for Td in SWEEP_T:
        i = np.arange(Td + 1, dtype=np.int64)
        ev = dict(x=(i % Wd).astype(np.uint16), y=(i % Hd).astype(np.uint16), t=i, p=(i & 1).astype(np.uint8))
        pos, _ = reference(ev, Wd, Hd, Td, NO_CUT)
        for ax, (name, dim) in enumerate((("x", Wd), ("y", Hd), ("t", Td))):
            src = (ev["x"], ev["y"], ev["t"])[ax].astype(np.int64)
            bad = pos[:, ax] != src
            pairs = np.unique(np.stack([src[bad], pos[bad, ax].astype(np.int64)], 1), axis=0).reshape(-1, 2)
            key = f"{name}{dim}"
            if key in exc:
                assert np.array_equal(exc[key], pairs), key
            exc[key] = pairs
        dims.append([Wd, Hd, Td])
        print(f"sweep W={Wd} H={Hd} T={Td}: x {int((pos[:, 0] != ev['x']).sum())}, y {int((pos[:, 1] != ev['y']).sum())}, "
              f"t {int((pos[:, 2] != ev['t']).sum())} values truncate below their input")
for key, pairs in exc.items():
    assert (pairs[:, 1] < pairs[:, 0]).all(), key
    out[f"sweep_{key}_in"] = pairs[:, 0].astype(np.int32)
    out[f"sweep_{key}_out"] = pairs[:, 1].astype(np.int32)
out["sweep_dims"] = np.array(dims, np.int64)
np.savez_compressed(HERE / "ingest_window_golden.npz", **out)
print("wrote", len(out), "arrays")
