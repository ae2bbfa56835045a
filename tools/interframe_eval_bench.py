"""The interframe evaluation (run_test_interframe's mAP per offset) on one synthetic DSEC-shaped recording, two routes in one
process, alternated over two rounds:

  device   InterframeEvaluation.add + compute: pair selection on the host, one SequenceDetector.detect over every window,
           dagr_interframe_targets + dagr_eval_pack_detections, one grouped dagr_evaluate_bbox launch.  Wall time split into
           pair selection, detection, targets + packing (including their small uploads), and evaluation.
  per-window  what a user does without it: the oracle's labels (oracle/ref_labels.py), one ground-truth dict per window,
           SequenceDetector.detect's per-window dicts, one DetectionBuffer per offset.  Its metrics are asserted equal to
           the device route's, float for float.

Recording: 60 s of raw 640x480 events (300 k events/s, clustered), frames and labels at 20 Hz (tests/interframe_cases.py:
about 10 moving boxes with stable track ids, births and deaths), dagr-s + ResNet-50 at 320x215 with raw_frames, 10
offsets.  A separate torch.profiler run gives the device time of the two new kernels' launches (their k_if_* / k_pk_*
kernels and the scans between them).  Card name, power limit and clocks are read in the same run.
Writes OUT/h100_interframe_eval.json (usage: python tools/interframe_eval_bench.py OUT)."""
import gc
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200 import labels as L
from dagr_b200.evaluation import DetectionBuffer
from dagr_b200.interframe import InterframeEvaluation
from dagr_b200.model.dagr import DAGR
from dagr_b200.sequence import SequenceDetector, interframe_windows
from dagr_b200.utils.args import default_args
from oracle import ref_labels as R
from tests import interframe_cases as IC
from tests.helpers import randomize_bn

W, H, SW, SH = 320, 215, 640, 480
SECONDS, RATE, STEPS, MIN_H, MIN_D = 60.0, 300_000, 10, 10, 15

if len(sys.argv) != 2:
    sys.exit("usage: python tools/interframe_eval_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def sync_ms(t0):
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


print("card (name, power limit, max SM clock, SM clock):", card(), flush=True)
torch.manual_seed(0)
model = randomize_bn(DAGR(default_args("s", batch_size=1, use_image=True, img_net="resnet50"), height=H, width=W).eval()).to(dev)
events, frame_t, tracks = IC.recording(SECONDS, 5, W, H, rate=RATE, sensor=(SW, SH), t0=4_000_000_000)
frames = torch.randint(0, 256, (len(frame_t), SH, SW, 3), generator=torch.Generator().manual_seed(5), dtype=torch.uint8).numpy()
print(f"recording: {len(events['t'])} events, {len(frame_t)} frames, {len(tracks)} label rows", flush=True)


def device_route():
    ev = InterframeEvaluation(model, IC.SOURCE, steps=STEPS, min_bbox_height=MIN_H, min_bbox_diag=MIN_D, sensor=(SW, SH),
                              raw_frames=True, max_windows=64)
    split = dict(targets_pack_ms=0.0)
    real = ev._launch

    def launch(rec, kept):                                  # the detections are complete before, the packed arrays after
        torch.cuda.synchronize()
        t = time.perf_counter()
        real(rec, kept)
        split["targets_pack_ms"] += sync_ms(t)

    ev._launch = launch
    gc.collect()
    gc.disable()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ev.add(events, frames, frame_t, tracks, sequence="synthetic")
    split["add_ms"] = sync_ms(t0)
    t1 = time.perf_counter()
    metrics = ev.compute()
    split["evaluate_ms"] = sync_ms(t1)
    split["total_ms"] = sync_ms(t0)
    gc.enable()
    t2 = time.perf_counter()
    L.pair_labels(tracks, frame_t, IC.SOURCE, W, H, 2, MIN_H, MIN_D)
    split["pair_selection_ms"] = (time.perf_counter() - t2) * 1e3
    split["detection_ms"] = split["add_ms"] - split["targets_pack_ms"] - split["pair_selection_ms"]
    split["windows"] = STEPS * ev.recordings[0]["P"]
    split["pairs"] = ev.recordings[0]["P"]
    split["gt_rows"] = int(ev.recordings[0]["gt_off"][-1])
    split["det_rows"] = int(ev.recordings[0]["dt_off"][-1])
    return metrics, split, ev


def per_window_route(offsets):
    gc.collect()
    gc.disable()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pairs, lab = R.recording_labels(tracks, frame_t, IC.SOURCE, W, H, 2, MIN_H, MIN_D)
    split = dict(labels_ms=(time.perf_counter() - t0) * 1e3)
    tb, te, fi = interframe_windows(frame_t[pairs[:, 0]], STEPS, 50_000)
    t1 = time.perf_counter()
    dets = SequenceDetector(model, sensor=(SW, SH), raw_frames=True, max_windows=64).detect(events, te, t_begin=tb, frames=frames,
                                                                                         frame_idx=pairs[fi, 0])
    split["detection_ms"] = sync_ms(t1)
    t2 = time.perf_counter()
    P, metrics = len(pairs), {}
    for g, n_us in enumerate(offsets):
        buf = DetectionBuffer(H, W, list(R.CLASSES))
        gts = []
        for p, (d0, d1) in enumerate(lab):
            b, lb = R.window_targets(d0, d1, int(frame_t[pairs[p, 0]]) + n_us, W, H, MIN_H, MIN_D, "numpy1")
            gts.append(dict(boxes=torch.from_numpy(b), labels=torch.from_numpy(lb)))
        buf.update(dets[g * P:(g + 1) * P], gts, "dsec")
        metrics[n_us] = buf.compute()
    split["targets_and_evaluate_ms"] = sync_ms(t2)
    split["total_ms"] = sync_ms(t0)
    gc.enable()
    return metrics, split


# warm-up on the first 3 s of the recording: module loads, graph captures, the image branch
warm = InterframeEvaluation(model, IC.SOURCE, steps=STEPS, min_bbox_height=MIN_H, min_bbox_diag=MIN_D, sensor=(SW, SH),
                            raw_frames=True, max_windows=64)
n_warm = int(np.searchsorted(frame_t, frame_t[0] + 3_000_000))
e_warm = int(np.searchsorted(events["t"], frame_t[n_warm]))
warm.add({k: v[:e_warm] for k, v in events.items()}, frames[:n_warm], frame_t[:n_warm],
         tracks[tracks["t"] < frame_t[n_warm]], sequence="warm")
warm.compute()
del warm

rounds, ev_last = [], None
for rnd in range(2):
    m_dev, s_dev, ev_last = device_route()
    m_pw, s_pw = per_window_route(ev_last.offsets)
    equal = all(m_dev[k] == m_pw[k] for k in m_pw) and list(m_dev) == list(m_pw)
    assert equal, (m_dev, m_pw)
    rounds.append(dict(round=rnd, device=s_dev, per_window=s_pw, equal=equal))
    print(f"[{rnd}] device {s_dev['total_ms']:.0f} ms (pairs {s_dev['pair_selection_ms']:.0f}, detection {s_dev['detection_ms']:.0f}, "
          f"targets+pack {s_dev['targets_pack_ms']:.1f}, evaluate {s_dev['evaluate_ms']:.1f}); per-window {s_pw['total_ms']:.0f} ms "
          f"(labels {s_pw['labels_ms']:.0f}, detection {s_pw['detection_ms']:.0f}, targets+evaluate {s_pw['targets_and_evaluate_ms']:.0f}); "
          f"equal {equal}", flush=True)

# device time of the two new kernels' launches (profiled on their own, after the timed rounds)
rec = ev_last.recordings[0]
from torch.profiler import ProfilerActivity, profile   # noqa: E402
real_launch = InterframeEvaluation._launch
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(10):
        real_launch(ev_last, rec, rec["P"])
    torch.cuda.synchronize()
kern = {}
for e in prof.key_averages():
    if e.key.startswith(("k_if_", "k_pk_", "k_scan_")):
        kern[e.key] = dict(calls=e.count, device_us_total=e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
per_call_us = sum(v["device_us_total"] for v in kern.values()) / 10
print(f"targets + packing kernels: {per_call_us:.1f} us of device time per recording ({rounds[-1]['device']['windows']} windows)")
print("card at end:", card(), flush=True)

out = dict(card_at_end=card(), shape=dict(model="dagr-s + resnet50", width=W, height=H, sensor=[SW, SH], seconds=SECONDS,
                                          rate_ev_s=RATE, frame_us=50_000, steps=STEPS, boxes=10),
           metrics={str(k): v for k, v in m_dev.items()},
           rounds=rounds, kernels=dict(per_recording_us=per_call_us, by_kernel=kern),
           note="wall times on one H100 with a host synchronise at the end of each part; detection is the same "
                "SequenceDetector call in both routes; kernels = torch.profiler device time of dagr_interframe_targets + "
                "dagr_eval_pack_detections (their kernels and scans) for the whole recording, averaged over 10 launches")
(out_dir / "h100_interframe_eval.json").write_text(json.dumps(out, indent=1))
print("wrote", out_dir / "h100_interframe_eval.json")
