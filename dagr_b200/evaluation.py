"""COCO detection metrics on the device: the reference's DetectionBuffer (src/dagr/utils/buffers.py:101-123) and
evaluate_detection (src/dagr/utils/coco_eval.py:64-94), without pycocotools or detectron2.

What the reference computes through its plumbing, and this module reproduces:
  - every box gets t = 0, so each image with at least one GT box is one COCO image (time_tol has no effect) and an image
    without GT contributes nothing, its detections included;
  - no detection in the kept images at all -> every metric is 0;
  - x, y, w = x2 - x1, h = y2 - y1 and the areas in float32, category = label + 1, the classes' categories only;
  - COCOeval('bbox') evaluate + accumulate with maxDets = 100 on the device (dagr_evaluate_bbox), then summarize's six
    AP figures with numpy on the small precision array, as pycocotools does.
There is no CPU path: without a CUDA device `compute` / `evaluate_detection` raise RuntimeError.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence

import numpy as np
import torch

from . import _lib
from .utils.buffers import compile as _compile

OUT_KEYS = ("AP", "AP_50", "AP_75", "AP_S", "AP_M", "AP_L")
# pycocotools Params.setDetParams: the float64 bits of these arrays are part of the metric (iou_thrs[7] = 0.8500000000000001)
IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]


def _params() -> _lib.EvalParams:
    p = _lib.EvalParams()
    p.iou_thrs[:] = IOU_THRS.tolist()
    p.rec_thrs[:] = REC_THRS.tolist()
    p.area_rng[:] = [float(v) for r in AREA_RNG for v in r]
    return p


def workspace_bytes(n_images: int, num_classes: int, n_gt: int, n_det: int) -> int:
    out = C.c_int64(0)
    _lib.check(_lib.load().dagr_eval_workspace_bytes(n_images, num_classes, n_gt, n_det, out), "dagr_eval_workspace_bytes")
    return out.value


def accumulate(gt_boxes_list: Sequence[Dict[str, torch.Tensor]], dt_boxes_list: Sequence[Dict[str, torch.Tensor]],
               num_classes: int, workspace: torch.Tensor = None):
    """COCOeval evaluate + accumulate of the images that have GT, on the device.  Returns (precision f64[10, 101, K, 4],
    recall f64[10, K, 4]) as CUDA tensors without synchronising, or None when those images hold no detection.
    `workspace`: a uint8 CUDA tensor of at least workspace_bytes(...) to run in (its contents do not matter); by default
    one is allocated."""
    pairs = [(g, d) for g, d in zip(gt_boxes_list, dt_boxes_list) if len(g["boxes"]) > 0]
    n_det = sum(len(d["boxes"]) for _, d in pairs)
    if n_det == 0:
        return None
    if not torch.cuda.is_available():
        raise RuntimeError("dagr_b200: detection evaluation runs on a CUDA device (there is no CPU path)")
    if workspace is not None and (not workspace.is_cuda or workspace.dtype != torch.uint8 or not workspace.is_contiguous()):
        raise ValueError("workspace must be a contiguous uint8 CUDA tensor")
    lib = _lib.load()
    dev = next((t.device for g, d in pairs for t in (g["boxes"], d["boxes"]) if t.is_cuda),
               workspace.device if workspace is not None else torch.device("cuda"))
    K, n = int(num_classes), len(pairs)

    def rows(key, dicts, dtype, width=None):
        parts = [d[key].to(dev, dtype).reshape(-1, width) if width else d[key].to(dev, dtype).reshape(-1) for d in dicts]
        return torch.cat(parts).contiguous()

    gts, dts = [g for g, _ in pairs], [d for _, d in pairs]
    gt_box, gt_lab = rows("boxes", gts, torch.float32, 4), rows("labels", gts, torch.int64)
    dt_box, dt_lab = rows("boxes", dts, torch.float32, 4), rows("labels", dts, torch.int64)
    dt_score = torch.cat([d["scores"].to(dev, torch.float32).reshape(-1) if "scores" in d else
                          torch.ones(len(d["boxes"]), dtype=torch.float32, device=dev) for d in dts])
    gt_off = torch.tensor(np.cumsum([0] + [len(g["boxes"]) for g in gts]), dtype=torch.int64).to(dev)
    dt_off = torch.tensor(np.cumsum([0] + [len(d["boxes"]) for d in dts]), dtype=torch.int64).to(dev)
    with torch.cuda.device(dev):
        need = workspace_bytes(n, K, len(gt_box), len(dt_box))
        if workspace is None:
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
        else:
            if workspace.device != dev or workspace.numel() < need:
                raise ValueError(f"workspace must be on {dev} and hold at least {need} bytes")
            ws = workspace
        precision = torch.empty((len(IOU_THRS), len(REC_THRS), K, len(AREA_RNG)), dtype=torch.float64, device=dev)
        recall = torch.empty((len(IOU_THRS), K, len(AREA_RNG)), dtype=torch.float64, device=dev)
        _lib.check(lib.dagr_evaluate_bbox(gt_box, gt_lab, gt_off, dt_box, dt_score, dt_lab, dt_off, n, K, len(gt_box), len(dt_box),
                                          _params(), ws, ws.numel(), precision, recall, _lib.stream_ptr()), "dagr_evaluate_bbox")
    return precision, recall


def summarize(precision: np.ndarray) -> Dict[str, float]:
    """COCOeval.summarize's stats[0:6] (maxDets = 100) from precision f64[10, 101, K, 4]: the mean of the entries > -1."""
    def one(iou_thr=None, area="all"):
        s = precision
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        s = s[:, :, :, [AREA_LBL.index(area)]]
        return -1.0 if len(s[s > -1]) == 0 else float(np.mean(s[s > -1]))
    return dict(zip(OUT_KEYS, (one(), one(.5), one(.75), one(area="small"), one(area="medium"), one(area="large"))))


def evaluate_detection(gt_boxes_list: List[Dict[str, torch.Tensor]], dt_boxes_list: List[Dict[str, torch.Tensor]],
                       classes=("car", "pedestrian"), height: int = 240, width: int = 304, time_tol: int = 50000) -> Dict[str, float]:
    """the reference's evaluate_detection: {'AP', 'AP_50', 'AP_75', 'AP_S', 'AP_M', 'AP_L'}.  height / width only label the
    COCO images and time_tol only matters for boxes with different times, so neither changes the result."""
    out = accumulate(gt_boxes_list, dt_boxes_list, len(classes)) if len(classes) > 0 else None
    if out is None:
        if len(classes) == 0 and any(len(d["boxes"]) for g, d in zip(gt_boxes_list, dt_boxes_list) if len(g["boxes"])):
            return {k: -1.0 for k in OUT_KEYS}                           # no category: every summary is empty
        return {k: 0.0 for k in OUT_KEYS}
    return summarize(out[0].cpu().numpy())


class DetectionBuffer:
    """the reference's DetectionBuffer: `update` collects per-image dicts (device tensors are kept as they are, host tensors
    are uploaded), `compute` evaluates them on the device, renames AP -> mAP and clears the buffer."""

    def __init__(self, height: int, width: int, classes: List[str]):
        self.height = height
        self.width = width
        self.classes = classes
        self.detections: List[Dict[str, torch.Tensor]] = []
        self.ground_truth: List[Dict[str, torch.Tensor]] = []

    @staticmethod
    def _to_device(dicts):
        if not torch.cuda.is_available():
            return list(dicts)                                           # compute() raises: there is no CPU path
        return [{k: v if v.is_cuda else v.cuda(non_blocking=True) for k, v in d.items()} for d in dicts]

    def compile(self, sequences, timestamps):
        cpu = lambda dicts: [{k: v.cpu() for k, v in d.items()} for d in dicts]
        return _compile(cpu(self.detections), sequences, timestamps), _compile(cpu(self.ground_truth), sequences, timestamps)

    def update(self, detections: List[Dict[str, torch.Tensor]], groundtruth: List[Dict[str, torch.Tensor]], dataset: str,
               height=None, width=None):
        self.detections.extend(self._to_device(detections))
        self.ground_truth.extend(self._to_device(groundtruth))

    def compute(self) -> Dict[str, float]:
        if not torch.cuda.is_available():
            raise RuntimeError("dagr_b200: detection evaluation runs on a CUDA device (there is no CPU path)")
        out = evaluate_detection(self.ground_truth, self.detections, height=self.height, width=self.width, classes=self.classes)
        out = {k.replace("AP", "mAP"): v for k, v in out.items()}
        self.detections.clear()
        self.ground_truth.clear()
        return out
