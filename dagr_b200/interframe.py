"""The reference's interframe evaluation (scripts/run_test_interframe.py) on the device: mAP at each offset after a frame.

    ev = InterframeEvaluation(model, source_classes, steps=10, span_us=50_000)
    ev.add(events, frames, frame_t, tracks, sequence="zurich_city_13_b")   # one recording; call in the dataset's order
    metrics = ev.compute()        # {n_us: {"mAP", "mAP_50", "mAP_75", "mAP_S", "mAP_M", "mAP_L"}}
    records = ev.detections()     # {sequence: records}, what the reference's save_detections writes

For each n_us = int(v) of np.linspace(0, span_us, steps), the reference runs the model on the window
[t_frame, t_frame + n_us) of every kept frame pair (i0, i1) -- with the image of frame i0 -- and scores it against the
pair's labels moved to t_frame + n_us by interpolate_tracks, after the test-time Crop and filter_small_bboxes.

How `add` runs: the pairs and their label tables come from labels.pair_labels on the host (once per recording); the
windows of the pairs' first frames (sequence.interframe_windows, offset-major, then pair) run through one
SequenceDetector.detect; dagr_interframe_targets interpolates, crops, filters and compacts the ground truth of every
window, and dagr_eval_pack_detections lays the detections out for the evaluation, dropping those of windows without ground
truth.  Both write category group * K + class, group = the offset's index, so `compute` scores every offset of every
recording in ONE dagr_evaluate_bbox call over steps * K categories: COCOeval matches per (image, category), a category
only sees its own offset's windows, and within an offset the windows keep the loader's order (recording, then pair), so the
stable score sort breaks ties as one evaluation per offset would.  `compute` reads back the per-window offsets once (for
the workspace size and the offsets without detections) and summarizes each offset's slice of the precision array.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List

import numpy as np
import torch

from . import _lib, evaluation, labels
from .sequence import SequenceDetector, interframe_windows
from .utils.buffers import records_from_device


class InterframeEvaluation:
    """mAP per offset after a frame over recordings added in the dataset's order.

    model: a DAGR model (events-only or image fusion) at the dataset's cropped resolution (DSEC: 320 x 215).
    source_classes: the recording's class names in class_id order (dsec_det's classes), mapped by labels.MAPPING onto
    labels.CLASSES.  min_bbox_height / min_bbox_diag: the dataset's size filters (run_test_interframe: 10 and 15), applied
    to the frame labels and again to each window's interpolated boxes.  scale: sensor pixels per model pixel of the labels.
    sensor / raw_frames: as SequenceDetector (raw camera events and frames; frame_t then in raw sensor time).
    reference_batch_size=b mirrors the reference loader's drop_last=True (run_test_interframe.py:69): the last
    len % b pairs of the whole dataset (all recordings added, in order) are neither run nor scored -- a quirk of the
    reference's numbers, not of the metric.  The default None keeps every pair.
    **sequence_kw: max_windows, max_events, p_is_01, device of the SequenceDetector."""

    def __init__(self, model, source_classes, steps: int = 10, span_us: int = 50_000, min_bbox_height=10, min_bbox_diag=15,
                 scale: int = 2, sensor=None, raw_frames: bool = False, reference_batch_size=None, **sequence_kw):
        if int(steps) < 1:
            raise ValueError(f"steps={steps} must be >= 1")
        if reference_batch_size is not None and int(reference_batch_size) < 1:
            raise ValueError(f"reference_batch_size={reference_batch_size} must be >= 1")
        self.detector = SequenceDetector(model, sensor=sensor, raw_frames=raw_frames, **sequence_kw)
        self.source_classes = list(source_classes)
        labels.compute_class_mapping(labels.CLASSES, self.source_classes)       # KeyError on a class the mapping lacks
        self.steps, self.span_us = int(steps), int(span_us)
        self.offsets = [int(n_us) for n_us in np.linspace(0, self.span_us, self.steps)]
        self.min_bbox_height, self.min_bbox_diag, self.scale = min_bbox_height, min_bbox_diag, int(scale)
        self.batch = None if reference_batch_size is None else int(reference_batch_size)
        self.K = len(labels.CLASSES)
        self.W, self.H, self.dev = self.detector.W, self.detector.H, self.detector.dev
        self.recordings: List[dict] = []
        self.last = None                    # (precision, recall) of the last compute(), categories g * K + class

    # ---- one recording -----------------------------------------------------------------------------------------------
    def add(self, events, frames, frame_t, tracks, sequence: str):
        """one recording: its events (SequenceDetector.detect's format), frames (None for an events-only model), the
        frames' timestamps, and its tracks (labels.pair_labels' format).  Bad input raises ValueError before device work."""
        ft = np.asarray(frame_t)
        if not self.detector.use_image and frames is not None:
            raise ValueError("frames are for image-fusion models; this model is events-only")
        if self.detector.use_image and (frames is None or len(frames) != len(ft)):
            raise ValueError(f"an image-fusion model needs one frame per frame time ({len(ft)})")
        pl = labels.pair_labels(tracks, ft, self.source_classes, self.W, self.H, self.scale, self.min_bbox_height, self.min_bbox_diag)
        rec = dict(sequence=str(sequence), labels=pl, P=len(pl))
        if len(pl):
            i0 = pl.pairs[:, 0]
            tb, te, fi = interframe_windows(pl.t[:, 0], self.steps, self.span_us)
            kw = dict(frames=frames, frame_idx=i0[fi]) if self.detector.use_image else {}
            self.detector.detect(events, te, t_begin=tb, **kw)
            det, ndet = self.detector.last
            dev = self.dev
            d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
            # the label tables, with one empty pair appended for the windows reference_batch_size drops
            rec.update(det=det, ndet=ndet, t_end=te, box0=d(pl.box0), box1=d(pl.box1), cls=d(pl.cls),
                       pair_off=d(np.concatenate([pl.off, pl.off[-1:]])), pair_t=d(np.concatenate([pl.t, pl.t[-1:]]).reshape(-1)),
                       win_t=d(te), win_group=d(np.repeat(np.arange(self.steps, dtype=np.int32), len(pl))))
            self._launch(rec, len(pl))
        self.recordings.append(rec)

    def _launch(self, rec, kept: int):
        """dagr_interframe_targets + dagr_eval_pack_detections of one recording, its first `kept` pairs scored"""
        lib, dev, P, G = _lib.load(), self.dev, rec["P"], self.steps
        pl = rec["labels"]
        pair = np.where(np.arange(P) < kept, np.arange(P), P)                  # P: the empty pair
        win_pair = torch.from_numpy(np.tile(pair, G).astype(np.int64)).to(dev)
        Q, L = G * P, len(pl.box0)
        R = G * int(pl.off[min(kept, P)])
        with torch.cuda.device(dev):
            ws_t, ws_p = C.c_int64(0), C.c_int64(0)
            _lib.check(lib.dagr_interframe_targets_workspace_bytes(Q, R, ws_t), "dagr_interframe_targets_workspace_bytes")
            _lib.check(lib.dagr_eval_pack_workspace_bytes(Q, ws_p), "dagr_eval_pack_workspace_bytes")
            ws = torch.empty(max(ws_t.value, ws_p.value), dtype=torch.uint8, device=dev)
            gt_box = torch.empty((R, 4), dtype=torch.float32, device=dev)
            gt_label = torch.empty(R, dtype=torch.int64, device=dev)
            gt_off = torch.empty(Q + 1, dtype=torch.int64, device=dev)
            _lib.check(lib.dagr_interframe_targets(
                rec["box0"], rec["box1"], rec["cls"], rec["pair_off"], rec["pair_t"], P + 1, L, win_pair, rec["win_t"],
                rec["win_group"], Q, self.K, self.W, self.H, float(self.min_bbox_height), float(self.min_bbox_diag), R, ws,
                ws.numel(), gt_box, gt_label, gt_off, _lib.stream_ptr()), "dagr_interframe_targets")
            det, ndet = rec["det"], rec["ndet"]
            A = det.shape[1]
            dt_box = torch.empty((Q * A, 4), dtype=torch.float32, device=dev)
            dt_score = torch.empty(Q * A, dtype=torch.float32, device=dev)
            dt_label = torch.empty(Q * A, dtype=torch.int64, device=dev)
            dt_off = torch.empty(Q + 1, dtype=torch.int64, device=dev)
            _lib.check(lib.dagr_eval_pack_detections(
                det, ndet, Q, A, rec["win_group"], gt_off, self.K, ws, ws.numel(), dt_box, dt_score, dt_label, dt_off,
                _lib.stream_ptr()), "dagr_eval_pack_detections")
        rec.update(kept=kept, gt_box=gt_box, gt_label=gt_label, gt_off=gt_off, dt_box=dt_box, dt_score=dt_score, dt_label=dt_label,
                   dt_off=dt_off)

    def _apply_batch(self):
        """reference_batch_size: the trailing len % b pairs of the dataset are not scored"""
        total = sum(r["P"] for r in self.recordings)
        drop = total % self.batch if self.batch else 0
        for r in reversed(self.recordings):
            keep = max(r["P"] - drop, 0)
            drop -= r["P"] - keep
            if r["P"] and keep != r.get("kept", r["P"]):
                self._launch(r, keep)

    # ---- results -----------------------------------------------------------------------------------------------------
    def compute(self) -> Dict[int, Dict[str, float]]:
        """{n_us: DetectionBuffer.compute's metrics of that offset}, over every recording added so far"""
        if self.dev.type != "cuda":
            raise RuntimeError("dagr_b200: the interframe evaluation runs on a CUDA device (there is no CPU path)")
        self._apply_batch()
        recs = [r for r in self.recordings if r["P"]]
        zero = {k.replace("AP", "mAP"): 0.0 for k in evaluation.OUT_KEYS}
        if not recs:
            return {n_us: dict(zero) for n_us in self.offsets}
        G, K = self.steps, self.K
        offs = torch.cat([torch.stack([r["gt_off"], r["dt_off"]]) for r in recs], dim=1).cpu().numpy()   # the one read-back
        n_gt, n_det, det_per_group = [], [], np.zeros(G, dtype=np.int64)
        at = 0
        for r in recs:
            Q = G * r["P"]
            go, do = offs[0, at:at + Q + 1], offs[1, at:at + Q + 1]
            n_gt.append(int(go[-1]))
            n_det.append(int(do[-1]))
            det_per_group += do[r["P"]::r["P"]] - do[:-1:r["P"]]
            at += Q + 1
        if sum(n_det) == 0:
            return {n_us: dict(zero) for n_us in self.offsets}
        dev = self.dev
        gb, db = np.cumsum([0] + n_gt), np.cumsum([0] + n_det)
        cat_off = lambda key, base: torch.cat([recs[0][key][:1]] + [r[key][1:] + int(b) for r, b in zip(recs, base)])
        gt_off, dt_off = cat_off("gt_off", gb), cat_off("dt_off", db)
        gt_box = torch.cat([r["gt_box"][:n] for r, n in zip(recs, n_gt)]).contiguous()
        gt_label = torch.cat([r["gt_label"][:n] for r, n in zip(recs, n_gt)])
        dt_box = torch.cat([r["dt_box"][:n] for r, n in zip(recs, n_det)]).contiguous()
        dt_score = torch.cat([r["dt_score"][:n] for r, n in zip(recs, n_det)])
        dt_label = torch.cat([r["dt_label"][:n] for r, n in zip(recs, n_det)])
        n_images = len(gt_off) - 1
        with torch.cuda.device(dev):
            need = evaluation.workspace_bytes(n_images, G * K, len(gt_box), len(dt_box))
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            precision = torch.empty((len(evaluation.IOU_THRS), len(evaluation.REC_THRS), G * K, len(evaluation.AREA_RNG)),
                                    dtype=torch.float64, device=dev)
            recall = torch.empty((len(evaluation.IOU_THRS), G * K, len(evaluation.AREA_RNG)), dtype=torch.float64, device=dev)
            _lib.check(_lib.load().dagr_evaluate_bbox(
                gt_box, gt_label, gt_off, dt_box, dt_score, dt_label, dt_off, n_images, G * K, len(gt_box), len(dt_box),
                evaluation._params(), ws, ws.numel(), precision, recall, _lib.stream_ptr()), "dagr_evaluate_bbox")
        self.last = (precision, recall)
        prec = precision.cpu().numpy()
        out = {}
        for g, n_us in enumerate(self.offsets):
            if det_per_group[g] == 0:                                   # evaluate_detection: no detection -> every metric 0
                out[n_us] = dict(zero)
            else:
                m = evaluation.summarize(prec[:, :, g * K:(g + 1) * K, :])
                out[n_us] = {k.replace("AP", "mAP"): v for k, v in m.items()}
        return out

    def detections(self) -> Dict[str, np.ndarray]:
        """{sequence: records (t, x, y, w, h, class_id, class_confidence)} of every scored window with t = t_frame + n_us:
        what the reference's save_detections writes, its windows listed offset-major, then recording, then pair, and each
        sequence sorted by t (stably: the reference's quicksort leaves the order of equal stamps unspecified)."""
        self._apply_batch()
        per_rec = []
        for r in self.recordings:
            if not r["P"] or not r["kept"]:                              # no pair, or every pair dropped: never run
                per_rec.append(None)
                continue
            recs = records_from_device(r["det"], r["ndet"], r["t_end"].tolist())
            per_rec.append([recs[g * r["P"]:g * r["P"] + r["kept"]] for g in range(self.steps)])
        seq: Dict[str, list] = {}
        for g in range(self.steps):
            for r, rr in zip(self.recordings, per_rec):
                if rr is not None:
                    seq.setdefault(r["sequence"], []).extend(rr[g])
        out = {}
        for s, parts in seq.items():
            a = np.concatenate(parts)
            out[s] = a[np.argsort(a["t"], kind="stable")]
        return out
