#!/usr/bin/env python
"""Generate tests/golden/frame_golden.npz from the REFERENCE's own camera-frame preparation (build container only):
`DSEC.preprocess_image` (src/dagr/data/dsec_data.py:149-154), the row crop and cv2.resize(INTER_CUBIC) every DSEC frame
goes through, run unmodified with the real OpenCV.

    DAGR_REFERENCE=/path/to/uzh-rpg/dagr python tests/golden/make_frame_golden.py

dsec_data.py imports torch_geometric, dsec_det and the reference's own data / visualisation modules at module level for
the rest of the dataset class; they are stubbed, and the method is called on a stub `self` carrying scale / height /
width.  Cases (frames are HWC u8 as the camera delivers them, outputs the method's [1, 3, H, W] u8):
  c0, c1  the DSEC shape, 640x480 -> 320x215 (scale 2, crop to 430 rows): ramps, and a checkerboard with 0 / 255 blocks
  c2..c5  small random frames at scales 1, 2, 3 and 4
  c6      a random frame 5 rows taller than scale * H (scale 2), so the crop matters
"""
import importlib.util
import os
import sys
import types
from pathlib import Path

import numpy as np


class _Stub(types.ModuleType):
    def __getattr__(self, name):                                     # any imported name: a placeholder class
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


if not os.environ.get("DAGR_REFERENCE"):
    sys.exit("set DAGR_REFERENCE to an uzh-rpg/dagr checkout")
SRC = Path(os.environ["DAGR_REFERENCE"]) / "src" / "dagr" / "data" / "dsec_data.py"
for name in ("torch_geometric", "torch_geometric.data", "dsec_det", "dsec_det.dataset", "dsec_det.io", "dsec_det.directory",
             "dagr", "dagr.data", "dagr.data.dsec_utils", "dagr.data.augment", "dagr.data.utils", "dagr.visualization",
             "dagr.visualization.bbox_viz", "dagr.visualization.event_viz"):
    sys.modules.setdefault(name, _Stub(name))
spec = importlib.util.spec_from_file_location("ref_dsec_data", SRC)
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)
import cv2                                                           # noqa: E402  (the one dsec_data.py just imported)


def run(image, height, width, scale):
    me = types.SimpleNamespace(scale=scale, height=height, width=width)
    return ref.DSEC.preprocess_image(me, image.copy()).numpy()


rng = np.random.default_rng(11)
yy, xx = np.mgrid[0:480, 0:640]
ramps = np.stack([(xx * 255) // 639, (yy * 255) // 479, (xx + 2 * yy) % 256], -1).astype(np.uint8)
checker = np.where(((yy // 7) + (xx // 5)) % 2 == 0, 255, 0).astype(np.uint8)
checker = np.stack([checker, 255 - checker, checker], -1)
checker[100:200, 300:420] = 0
checker[250:330, 40:260] = 255
checker[400:480, 500:640] = (255, 0, 255)
cases = [(ramps, 215, 320, 2), (checker, 215, 320, 2)]
for s, (h, w) in zip((1, 2, 3, 4), ((9, 13), (11, 17), (7, 10), (6, 8))):
    cases.append((rng.integers(0, 256, (s * h, s * w, 3), dtype=np.uint8), h, w, s))
cases.append((rng.integers(0, 256, (2 * 12 + 5, 2 * 15, 3), dtype=np.uint8), 12, 15, 2))

out = {}
for i, (img, h, w, s) in enumerate(cases):
    out[f"c{i}_in"] = img
    out[f"c{i}_out"] = run(img, h, w, s)
    out[f"c{i}_geom"] = np.array([h, w, s])
out["cases"] = np.array(len(cases))
out["cv2_version"] = np.array(cv2.__version__)
dst = Path(__file__).parent / "frame_golden.npz"
np.savez_compressed(dst, **out)
print("wrote", dst, dst.stat().st_size, "bytes,", len(cases), "cases, cv2", cv2.__version__)
