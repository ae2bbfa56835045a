"""Host-side detection records (SURVEY 8(f) rank 2): what the reference does with the model's output on the CPU.

Only the record format is in scope (the evaluation harness around it is not, SURVEY section 2, #7):
  src/dagr/utils/buffers.py:46-76    bbox_t_to_ndarray / compile  (record dtype t,x,y,w,h,class_id[,class_confidence])
  scripts/run_test_interframe.py:21-45  to_npy / save_detections
plus `records_from_device`, which turns the batched device output of `Engine.postprocess` (det [B,A,6], ndet [B])
into one record array per image with a single device->host copy (the reference loops over images and tensors).
COCO evaluation (DetectionBuffer.compute, src/dagr/utils/coco_eval.py) runs on the device in dagr_b200.evaluation.
"""
from __future__ import annotations

from pathlib import Path
from typing import Dict, List, Sequence

import numpy as np
import torch

from ..data import format_data  # noqa: F401  (re-exported like the reference module)

_REC = [("t", "<u8"), ("x", "<f4"), ("y", "<f4"), ("w", "<f4"), ("h", "<f4"), ("class_id", "u1")]
_REC_CONF = _REC + [("class_confidence", "<f4")]


def _records(t, boxes: np.ndarray, labels: np.ndarray, scores=None) -> np.ndarray:
    rec = np.zeros(shape=(len(boxes),), dtype=_REC if scores is None else _REC_CONF)
    rec["t"] = t
    rec["x"], rec["y"] = boxes[:, 0], boxes[:, 1]
    rec["w"], rec["h"] = boxes[:, 2] - boxes[:, 0], boxes[:, 3] - boxes[:, 1]
    rec["class_id"] = labels
    if scores is not None:
        rec["class_confidence"] = scores
    return rec


def bbox_t_to_ndarray(bbox: Dict[str, torch.Tensor], t) -> np.ndarray:
    """one image: dict(boxes xyxy, labels[, scores]) on the CPU -> structured records; a dict with three entries is a
    detection (gets class_confidence), one with two a ground-truth box set."""
    scores = bbox["scores"].numpy() if len(bbox) == 3 else None
    return _records(t, bbox["boxes"].numpy(), bbox["labels"].numpy(), scores)


def compile(detections, sequences, timestamps):  # noqa: A001  (name kept from the reference)
    per_seq: Dict[str, list] = {}
    for det, s, t in zip(detections, sequences, timestamps):
        per_seq.setdefault(s, []).append(bbox_t_to_ndarray(det, t))
    return {k: np.concatenate(v) for k, v in per_seq.items() if len(v) > 0}


# ---- scripts/run_test_interframe.py:21-45 ---------------------------------------------------------------------------
def to_npy(detections) -> np.ndarray:
    """dict(boxes, labels, scores, t) of one image -> records with class_confidence (w, h derived from the stored x, y)."""
    boxes = np.asarray(detections["boxes"], dtype=np.float32).reshape(-1, 4)
    rec = np.zeros(shape=(len(boxes),), dtype=np.dtype(_REC_CONF))
    rec["t"] = detections["t"]
    rec["x"], rec["y"] = boxes[:, 0], boxes[:, 1]
    rec["w"], rec["h"] = boxes[:, 2] - rec["x"], boxes[:, 3] - rec["y"]
    rec["class_id"] = np.asarray(detections["labels"])
    rec["class_confidence"] = np.asarray(detections["scores"])
    return rec


def save_detections(directory, detections: Sequence[dict]):
    """groups by d['sequence'], sorts each sequence by t and writes detections_<sequence>.npy; returns the arrays."""
    per_seq: Dict[str, np.ndarray] = {}
    for d in detections:
        s, rec = d["sequence"], to_npy(d)
        per_seq[s] = rec if s not in per_seq else np.concatenate([per_seq[s], rec])
    out = {}
    for s, rec in per_seq.items():
        rec = rec[rec["t"].argsort()]
        np.save(Path(directory) / f"detections_{s}.npy", rec)
        out[s] = rec
    return out


# ---- batched device output -> records ------------------------------------------------------------------------------
def records_from_device(det: torch.Tensor, ndet: torch.Tensor, timestamps: Sequence[int]) -> List[np.ndarray]:
    """det float32[B,A,6] = (x1,y1,x2,y2,score,label) sorted by score, ndet int32[B] (Engine.postprocess / the batched
    NMS kernel) -> one record array per image, with ONE device->host copy for the whole batch."""
    B, A, _ = det.shape
    host = torch.cat([det.reshape(B, -1), ndet.reshape(B, 1).to(det.dtype)], dim=1).cpu().numpy()
    out = []
    for b in range(B):
        n = int(host[b, -1])
        d = host[b, : A * 6].reshape(A, 6)[:n]
        out.append(_records(timestamps[b], d[:, :4], d[:, 5].astype(np.uint8), d[:, 4]))
    return out
