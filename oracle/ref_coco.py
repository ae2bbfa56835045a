"""numpy restatement of pycocotools 2.0's COCO / loadRes / COCOeval for 'bbox' (evaluate, accumulate, summarize), the
checker of dagr_b200.evaluation.  `COCO` and `COCOeval` stand in for pycocotools.coco.COCO and
detectron2.evaluation.fast_eval_api.COCOeval_opt (its C++ port): the same attributes and calls the reference's
coco_eval.py uses, with the float widths of that path (bbox entries and areas as the float32 values they arrive as,
IoU in double).  Crowd GT, segm / keypoints and the AR stats are not restated (iscrowd is always False there)."""
from __future__ import annotations

import copy

import numpy as np


class COCO:
    def __init__(self):
        self.dataset, self.anns, self.imgs, self.cats = {}, {}, {}, {}

    def createIndex(self):
        self.anns = {a["id"]: a for a in self.dataset.get("annotations", [])}
        self.imgs = {im["id"]: im for im in self.dataset.get("images", [])}
        self.cats = {c["id"]: c for c in self.dataset.get("categories", [])}

    def getCatIds(self):
        return [c["id"] for c in self.dataset.get("categories", [])]

    def getImgIds(self):
        return list(self.imgs.keys())

    def loadRes(self, anns):
        res = COCO()
        res.dataset["images"] = list(self.dataset["images"])
        assert isinstance(anns, list)
        assert set(a["image_id"] for a in anns) <= set(self.getImgIds())
        res.dataset["categories"] = copy.deepcopy(self.dataset["categories"])
        for k, ann in enumerate(anns):
            bb = ann["bbox"]
            ann["area"] = bb[2] * bb[3]                      # float32 scalars -> float32 product
            ann["id"] = k + 1
            ann["iscrowd"] = 0
        res.dataset["annotations"] = anns
        res.createIndex()
        return res


def bb_iou(d: np.ndarray, g: np.ndarray) -> np.ndarray:
    """maskApi.c bbIou with iscrowd = 0: d [m, 4], g [n, 4] float64 xywh -> [m, n]"""
    out = np.zeros((len(d), len(g)))
    for j in range(len(g)):
        gx, gy, gw, gh = (float(v) for v in g[j])
        ga = gw * gh
        for i in range(len(d)):
            dx, dy, dw, dh = (float(v) for v in d[i])
            w = min(dw + dx, gw + gx) - max(dx, gx)
            if w <= 0:
                continue
            h = min(dh + dy, gh + gy) - max(dy, gy)
            if h <= 0:
                continue
            inter = w * h
            out[i, j] = inter / (dw * dh + ga - inter)
    return out


class Params:
    def __init__(self):
        self.imgIds, self.catIds = [], []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [1, 10, 100]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ["all", "small", "medium", "large"]
        self.useCats = 1


def _order(scores) -> np.ndarray:
    return np.argsort([-s for s in scores], kind="mergesort")


class COCOeval:
    def __init__(self, cocoGt, cocoDt, iouType="bbox"):
        assert iouType == "bbox"
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.params = Params()
        self.params.imgIds = sorted(cocoGt.getImgIds())
        self.params.catIds = sorted(cocoGt.getCatIds())
        self.eval, self.stats = {}, []

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        gts, dts, imgs, cats = {}, {}, set(p.imgIds), set(p.catIds)
        for a in self.cocoGt.dataset["annotations"]:
            if a["image_id"] in imgs and a["category_id"] in cats:
                a["ignore"] = bool(a.get("iscrowd", 0))
                gts.setdefault((a["image_id"], a["category_id"]), []).append(a)
        for a in self.cocoDt.dataset["annotations"]:
            if a["image_id"] in imgs and a["category_id"] in cats:
                dts.setdefault((a["image_id"], a["category_id"]), []).append(a)
        self._gts, self._dts = gts, dts
        self.ious = {(i, c): self.computeIoU(i, c) for i in p.imgIds for c in p.catIds}
        maxDet = p.maxDets[-1]
        self.evalImgs = [self.evaluateImg(i, c, a, maxDet) for c in p.catIds for a in p.areaRng for i in p.imgIds]

    def computeIoU(self, imgId, catId):
        gt, dt = self._gts.get((imgId, catId), []), self._dts.get((imgId, catId), [])
        if len(gt) == 0 and len(dt) == 0:
            return []
        dt = [dt[i] for i in _order([d["score"] for d in dt])][:self.params.maxDets[-1]]
        if len(gt) == 0 or len(dt) == 0:
            return []
        return bb_iou(np.array([d["bbox"] for d in dt], dtype=np.double), np.array([g["bbox"] for g in gt], dtype=np.double))

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        p = self.params
        gt, dt = self._gts.get((imgId, catId), []), self._dts.get((imgId, catId), [])
        if len(gt) == 0 and len(dt) == 0:
            return None
        ign = [1 if (g["ignore"] or g["area"] < aRng[0] or g["area"] > aRng[1]) else 0 for g in gt]
        gtind = np.argsort(ign, kind="mergesort")
        gt = [gt[i] for i in gtind]
        gtIg = np.array([ign[i] for i in gtind])
        dt = [dt[i] for i in _order([d["score"] for d in dt])[0:maxDet]]
        ious = self.ious[imgId, catId]
        ious = ious[:, gtind] if len(ious) > 0 else ious
        T, G, D = len(p.iouThrs), len(gt), len(dt)
        gtm, dtm = np.zeros((T, G)), np.zeros((T, D))
        dtIg = np.zeros((T, D))
        if len(ious) != 0:
            for tind, t in enumerate(p.iouThrs):
                for dind in range(D):
                    iou, m = min([t, 1 - 1e-10]), -1
                    for gind in range(G):
                        if gtm[tind, gind] > 0:
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou, m = ious[dind, gind], gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = gt[m]["id"]
                    gtm[tind, m] = dt[dind]["id"]
        a = np.array([d["area"] < aRng[0] or d["area"] > aRng[1] for d in dt]).reshape((1, D))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {"dtMatches": dtm, "dtScores": [d["score"] for d in dt], "gtIgnore": gtIg, "dtIgnore": dtIg}

    def accumulate(self):
        p = self.params
        T, R, K, A, M = len(p.iouThrs), len(p.recThrs), len(p.catIds), len(p.areaRng), len(p.maxDets)
        precision, recall = -np.ones((T, R, K, A, M)), -np.ones((T, K, A, M))
        I = len(p.imgIds)
        for k in range(K):
            for a in range(A):
                for m, maxDet in enumerate(p.maxDets):
                    E = [e for e in self.evalImgs[k * A * I + a * I:k * A * I + a * I + I] if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e["dtScores"][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind="mergesort")
                    dtm = np.concatenate([e["dtMatches"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e["dtIgnore"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e["gtIgnore"] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        nd = len(tp)
                        rc = tp / npig
                        pr = (tp / (fp + tp + np.spacing(1))).tolist()
                        q = np.zeros((R,)).tolist()
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        for ri, pi in enumerate(np.searchsorted(rc, p.recThrs, side="left")):
                            if pi >= nd:
                                break
                            q[ri] = pr[pi]
                        precision[t, :, k, a, m] = np.array(q)
        self.eval = {"precision": precision, "recall": recall}

    def summarize(self):
        p = self.params

        def one(iouThr=None, areaRng="all", maxDets=100):
            aind = [i for i, r in enumerate(p.areaRngLbl) if r == areaRng]
            mind = [i for i, m in enumerate(p.maxDets) if m == maxDets]
            s = self.eval["precision"]
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, :, aind, mind]
            return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        stats = np.zeros((12,))
        stats[0], stats[1], stats[2] = one(), one(.5), one(.75)
        stats[3], stats[4], stats[5] = one(areaRng="small"), one(areaRng="medium"), one(areaRng="large")
        self.stats = stats


# ---- the reference's plumbing (coco_eval.py), restated for dicts of tensors --------------------------------------------
def to_records(d):
    """_to_prophesee: float32 x, y, w = x2 - x1, h = y2 - y1, uint32 class id, float32 confidence (ones without scores)"""
    b = d["boxes"].cpu().numpy().reshape(-1, 4)
    w, h = (b[:, 2] - b[:, 0]).astype(np.float32), (b[:, 3] - b[:, 1]).astype(np.float32)
    lab = d["labels"].cpu().numpy().astype(np.uint32)
    conf = d["scores"].cpu().numpy().astype(np.float32) if "scores" in d else np.ones(len(b), dtype=np.float32)
    return b[:, 0].astype(np.float32), b[:, 1].astype(np.float32), w, h, lab, conf


def evaluate_lists(gt_list, dt_list, num_classes: int):
    """COCOeval over the images with GT (image ids 1..n), as the reference builds it.  Returns the COCOeval object
    (eval['precision'][..., 2] is the maxDets = 100 slice), or None when those images hold no detection."""
    images, anns, results = [], [], []
    for g, d in zip(gt_list, dt_list):
        if len(g["boxes"]) == 0:
            continue
        im = len(images) + 1
        images.append({"id": im})
        for x, y, w, h, c, _ in zip(*to_records(g)):
            anns.append({"area": float(w * h), "iscrowd": False, "image_id": im, "bbox": [x, y, w, h],
                         "category_id": int(c) + 1, "id": len(anns) + 1})
        for x, y, w, h, c, s in zip(*to_records(d)):
            results.append({"image_id": im, "category_id": int(c) + 1, "score": float(s), "bbox": [x, y, w, h]})
    if not results:
        return None
    gt = COCO()
    gt.dataset = {"images": images, "annotations": anns, "categories": [{"id": k + 1} for k in range(num_classes)]}
    gt.createIndex()
    ev = COCOeval(gt, gt.loadRes(results), "bbox")
    ev.params.imgIds = np.arange(1, len(images) + 1, dtype=int)
    ev.evaluate()
    ev.accumulate()
    ev.summarize()
    return ev
