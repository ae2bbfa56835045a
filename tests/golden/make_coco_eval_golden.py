#!/usr/bin/env python
"""Generate tests/golden/coco_eval_golden.npz from the REFERENCE's own src/dagr/utils/buffers.py and coco_eval.py
(build container only, both unmodified).  The third-party modules coco_eval imports -- pycocotools.coco.COCO and
detectron2.evaluation.fast_eval_api.COCOeval_opt -- are stood in for by oracle/ref_coco.py, so the fixture pins the
reference's plumbing around COCOeval: t = 0 matching, images without GT dropped, class_id + 1, the AP -> mAP renaming and
the zero dict.

    DAGR_REFERENCE=/path/to/uzh-rpg/dagr python tests/golden/make_coco_eval_golden.py
"""
import importlib.util
import os
import sys
import types
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle import ref_coco  # noqa: E402

REF = Path(os.environ["DAGR_REFERENCE"]) / "src" / "dagr" / "utils"
for name, attrs in (("pycocotools", {}), ("pycocotools.coco", {"COCO": ref_coco.COCO}), ("detectron2", {}),
                    ("detectron2.evaluation", {}), ("detectron2.evaluation.fast_eval_api", {"COCOeval_opt": ref_coco.COCOeval})):
    m = types.ModuleType(name)
    m.__path__ = []
    m.__dict__.update(attrs)
    sys.modules[name] = m
for name, path in (("refdagr", []), ("refdagr.utils", [str(REF)])):
    m = types.ModuleType(name)
    m.__path__ = path
    sys.modules[name] = m
for mod in ("coco_eval", "buffers"):
    spec = importlib.util.spec_from_file_location(f"refdagr.utils.{mod}", REF / f"{mod}.py")
    ref = importlib.util.module_from_spec(spec)
    sys.modules[f"refdagr.utils.{mod}"] = ref
    spec.loader.exec_module(ref)
buffers = sys.modules["refdagr.utils.buffers"]


def case(g, n_images, K, label_hi):
    """seeded images: a few GT boxes, detections near them (jittered, so IoUs spread over the thresholds) plus clutter;
    some images without GT, some without detections, labels up to label_hi - 1 (>= K: outside the classes)"""
    dets, gts = [], []
    for i in range(n_images):
        ng = 0 if i % 7 == 3 else int(torch.randint(1, 6, (1,), generator=g))
        xy = torch.rand(ng, 2, generator=g) * 400
        wh = torch.rand(ng, 2, generator=g) * 150 + 2
        gb = torch.cat([xy, xy + wh], 1)
        gl = torch.randint(0, label_hi, (ng,), generator=g)
        nd = 0 if i % 5 == 4 else int(torch.randint(0, 12, (1,), generator=g))
        src = torch.randint(0, max(ng, 1), (nd,), generator=g)
        base = gb[src] if ng else torch.rand(nd, 4, generator=g) * 300
        jit = (torch.rand(nd, 4, generator=g) - 0.5) * 30
        db = base + jit
        db = torch.cat([torch.minimum(db[:, :2], db[:, 2:]), torch.maximum(db[:, :2], db[:, 2:])], 1)
        dl = gl[src] if ng else torch.randint(0, label_hi, (nd,), generator=g)
        flip = torch.rand(nd, generator=g) < 0.15
        dl = torch.where(flip, torch.randint(0, label_hi, (nd,), generator=g), dl)
        sc = torch.round(torch.rand(nd, generator=g) * 20) / 20            # coarse scores: ties inside and across images
        gts.append(dict(boxes=gb, labels=gl))
        dets.append(dict(boxes=db, scores=sc, labels=dl))
    return dets, gts


out = {}
g = torch.Generator().manual_seed(11)
cases = {"k2": (case(g, 60, 2, 3), ("car", "pedestrian")),
         "k5": (case(g, 40, 5, 5), tuple(f"c{k}" for k in range(5))),
         "nodet": (([dict(boxes=torch.zeros(0, 4), scores=torch.zeros(0), labels=torch.zeros(0, dtype=torch.long))] * 3,
                    [dict(boxes=torch.tensor([[1., 2., 40., 50.]]), labels=torch.tensor([0]))] * 3), ("car", "pedestrian")),
         "nogt": (([dict(boxes=torch.tensor([[1., 2., 40., 50.]]), scores=torch.tensor([.9]), labels=torch.tensor([0]))] * 2,
                   [dict(boxes=torch.zeros(0, 4), labels=torch.zeros(0, dtype=torch.long))] * 2), ("car", "pedestrian"))}
for name, ((dets, gts), classes) in cases.items():
    for i, (d, gt) in enumerate(zip(dets, gts)):
        for k, v in d.items():
            out[f"{name}_det{i}_{k}"] = v.numpy().copy()
        for k, v in gt.items():
            out[f"{name}_gt{i}_{k}"] = v.numpy().copy()
    out[f"{name}_n"] = np.array(len(dets))
    out[f"{name}_K"] = np.array(len(classes))
    buf = buffers.DetectionBuffer(height=480, width=640, classes=list(classes))
    half = len(dets) // 2
    for lo, hi in ((0, half), (half, len(dets))):
        buf.update([{k: v.clone() for k, v in d.items()} for d in dets[lo:hi]],
                   [{k: v.clone() for k, v in d.items()} for d in gts[lo:hi]], "dsec")
    res = buf.compute()
    out[f"{name}_keys"] = np.array(sorted(res))
    out[f"{name}_stats"] = np.array([float(res[k]) for k in sorted(res)])
np.savez_compressed(Path(__file__).parent / "coco_eval_golden.npz", **out)
print("wrote", len(out), "arrays", {n: out[f"{n}_stats"].tolist() for n in cases})
