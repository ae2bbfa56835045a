#!/usr/bin/env python
"""Time DetectionBuffer.compute() (COCO bbox mAP on the device) on a DSEC-shaped workload and write OUT/h100_eval.json.

Workload: 2 classes, 0..175 detections per image (Engine.postprocess keeps at most A = 175 boxes at 640x480), 1..6 GT
boxes per image, detections jittered around the GTs plus clutter, scores with ties; 10k and 100k images held as CUDA
tensors (the DetectionBuffer state after `update` with model outputs).  compute() is timed end to end -- packing, the
kernels, the copy of the precision array and numpy's summarize -- by the host clock around the call, which ends in a
device synchronise (the copy of the precision array), after warm-up.
The restated COCOeval (oracle/ref_coco.py, pure numpy / Python, not pycocotools) is timed on the host on a small set.

    python tools/eval_bench.py OUT
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from dagr_b200 import evaluation  # noqa: E402


def workload(n_images, seed, device):
    g = torch.Generator().manual_seed(seed)
    ng = torch.randint(1, 7, (n_images,), generator=g)
    nd = torch.randint(0, 176, (n_images,), generator=g)
    G, D = int(ng.sum()), int(nd.sum())
    xy = torch.rand(G, 2, generator=g) * 560
    gb = torch.cat([xy, xy + torch.rand(G, 2, generator=g) * 120 + 4], 1)
    gl = torch.randint(0, 2, (G, ), generator=g)
    img_of_gt = torch.repeat_interleave(torch.arange(n_images), ng)
    gt_start = torch.cumsum(ng, 0) - ng
    img_of_dt = torch.repeat_interleave(torch.arange(n_images), nd)
    src = gt_start[img_of_dt] + (torch.rand(D, generator=g) * ng[img_of_dt]).long()
    db = gb[src] + torch.randn(D, 4, generator=g) * 6
    clutter = torch.rand(D, generator=g) < 0.5
    cxy = torch.rand(D, 2, generator=g) * 560
    db[clutter] = torch.cat([cxy, cxy + torch.rand(D, 2, generator=g) * 80 + 4], 1)[clutter]
    dl = torch.where(clutter, torch.randint(0, 2, (D,), generator=g), gl[src])
    sc = torch.round(torch.rand(D, generator=g) * 1000) / 1000
    assert int(img_of_gt[-1]) == n_images - 1
    gb, gl, db, dl, sc = (t.to(device) for t in (gb, gl, db, dl, sc))
    gts = [dict(boxes=b, labels=l) for b, l in zip(gb.split(ng.tolist()), gl.split(ng.tolist()))]
    dts = [dict(boxes=b, scores=s, labels=l) for b, s, l in zip(db.split(nd.tolist()), sc.split(nd.tolist()), dl.split(nd.tolist()))]
    return gts, dts, D


def time_compute(gts, dts, reps):
    ms = []
    for _ in range(reps):
        buf = evaluation.DetectionBuffer(480, 640, ["car", "pedestrian"])
        buf.update(dts, gts, "dsec")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = buf.compute()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return sorted(ms), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", help="directory that receives h100_eval.json")
    ap.add_argument("--sizes", default="10000,100000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle_images", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "eval_bench measures the device path: it needs a CUDA device"
    dev = torch.device("cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    out = {"gpu": q, "workload": "2 classes, 0..175 detections and 1..6 GT per image, CUDA tensors", "rows": []}
    warm_g, warm_d, _ = workload(2000, 1, dev)
    time_compute(warm_g, warm_d, 2)
    for n in (int(s) for s in a.sizes.split(",")):
        gts, dts, D = workload(n, n, dev)
        ms, res = time_compute(gts, dts, a.reps)
        row = {"images": n, "detections": D, "compute_ms_median": ms[len(ms) // 2], "compute_ms_min": ms[0], "mAP": res["mAP"]}
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
    from oracle import ref_coco
    gts, dts, D = workload(a.oracle_images, 7, torch.device("cpu"))
    t0 = time.perf_counter()
    ev = ref_coco.evaluate_lists(gts, dts, 2)
    host_s = time.perf_counter() - t0
    dev_res = evaluation.evaluate_detection([{k: v.to(dev) for k, v in x.items()} for x in gts],
                                            [{k: v.to(dev) for k, v in x.items()} for x in dts])
    out["oracle"] = {"what": "restated COCOeval in numpy / Python (oracle/ref_coco.py), host, not pycocotools",
                     "images": a.oracle_images, "detections": D, "seconds": host_s,
                     "stats_equal_device": [dev_res[k] for k in evaluation.OUT_KEYS] == ev.stats[:6].tolist()}
    print(json.dumps(out["oracle"]), flush=True)
    Path(a.out).mkdir(parents=True, exist_ok=True)
    (Path(a.out) / "h100_eval.json").write_text(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
