"""Interframe windows on live hybrid cameras (since_frame=True) against the sliding window, in one process: config 3's model
(dagr-s + ResNet-50, 640x480) on S = 1 and 8 copies of config 5's stream (1 Mevents/s per camera in 1 ms chunks, window_us =
50 ms, 2 s of stream), a new frame every 50 ms of stream time per camera, camera s's frames offset by s * 50 / S ms, never
waited for.  S = 1 runs FusionStreamingDetector, S = 8 FusionMultiStreamDetector; for each S the sliding and since_frame
routes alternate, two rounds.  Per run: step latency p50 / p99 (host, submit to detections on the host), device time p50
(CUDA events around the step), mean live events per step and camera, frame-to-first-use p50 (all cameras pooled).  Then the
device time of the since_frame step's extra work alone -- the D2D copy of the control blocks and the second push -- as 200
copies captured in one CUDA graph, per replay / 200.
Writes OUT/h100_interframe_stream.json (usage: python tools/interframe_stream_bench.py OUT)."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200.streaming import (FusionMultiStreamDetector, FusionStreamingDetector, _bench_setup, _dist, _FrameFeed,
                                 _timed_steps)

W, H = 640, 480
RATE, CHUNK, WINDOW, FRAME, SECONDS = 1_000_000, 1000, 50_000, 50_000, 2.0
STREAMS = (1, 8)
if len(sys.argv) != 2:
    sys.exit("usage: python tools/interframe_stream_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")


def smi(q):
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


card = smi("name,power.limit,clocks.max.sm,clocks.sm")
print("card (name, power limit, max SM clock, SM clock):", card, flush=True)
model, _, _, _ = _bench_setup(dev, None, "s", W, H, 1, RATE, CHUNK, WINDOW, 0.0, "uniform", use_image=True, img_net="resnet50")
setups = {S: _bench_setup(dev, model, "s", W, H, S, RATE, CHUNK, WINDOW, SECONDS, "uniform")[1:] for S in STREAMS}


class _Feed(_FrameFeed):
    """the benchmarks' frame feed, also recording each timed step's live events per camera."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.live = []

    def stepped(self, t1):
        super().stepped(t1)
        d = self.det
        self.live.append(np.mean([d._state(s)["live"] for s in range(d.S)]))


def run(S, since_frame):
    evs, bounds, max_chunk = setups[S]
    kw = dict(window_us=WINDOW, max_chunk=max_chunk, since_frame=since_frame)
    if S == 1:
        det = FusionStreamingDetector(model, **kw)
        submit, set_frame = (lambda c, te: det.submit(*c[0], te[0])), (lambda s, image, t_us: det.set_frame(image, t_us=t_us))
    else:
        det = FusionMultiStreamDetector(model, streams=S, **kw)
        submit, set_frame = det.submit, det.set_frame
    offset = [(s * FRAME // S) // CHUNK * CHUNK for s in range(S)]
    frames = _Feed(det, set_frame, FRAME, CHUNK, offset)
    lat, dev_ms, nev = _timed_steps(det, submit, evs, bounds, CHUNK, WINDOW, frames)
    first = [v for cam in frames.first_use for v in cam]
    r = dict(streams=S, since_frame=since_frame, steps=len(lat), stage_bytes=det.stage_bytes, graphs=len(det.graphs),
             latency_ms=_dist(lat), device_ms=_dist(dev_ms), live_events_mean=float(np.mean(frames.live)),
             events_per_step=float(np.mean(nev)), frame_to_first_use_ms=_dist(first),
             overflow=any(det._state(s)["overflow"] for s in range(S)))
    print(f"S = {S} {'since_frame' if since_frame else 'sliding    '}: p50 {r['latency_ms']['p50']:.3f} p99 {r['latency_ms']['p99']:.3f} ms, "
          f"device p50 {r['device_ms']['p50']:.3f} ms, live {r['live_events_mean']:.0f}, first use p50 "
          f"{r['frame_to_first_use_ms'].get('p50', float('nan')):.2f} ms", flush=True)
    return r, det


def extra_work_us(det, n=200):
    """device time of the since_frame step's extra work (control-block copy + second push) per step, from n copies
    captured in one graph (replayed after the run: the window is already cut, so it evicts nothing)."""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(det.stream):
        det._ctl_rows[1].copy_(det.ctl)
        det._push(det._cut_d, 1)                                      # warm
        det.stream.synchronize()
        with torch.cuda.graph(g, stream=det.stream):
            for _ in range(n):
                det._ctl_rows[1].copy_(det.ctl)
                det._push(det._cut_d, 1)
        out = []
        for _ in range(10):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(det.stream)
            g.replay()
            e1.record(det.stream)
            e1.synchronize()
            out.append(e0.elapsed_time(e1) * 1e3 / n)
    return sorted(out)


runs, extra = [], {}
for rnd in range(2):
    for S in STREAMS:
        for since in ((False, True) if rnd == 0 else (True, False)):
            r, det = run(S, since)
            runs.append(dict(round=rnd, **r))
            if since and rnd == 1:
                v = extra_work_us(det)
                extra[str(S)] = dict(median_us=v[len(v) // 2], min_us=v[0], max_us=v[-1])
                print(f"S = {S}: control-block copy + second push {v[len(v) // 2]:.2f} us per step (median of 10)", flush=True)
            del det
            torch.cuda.empty_cache()

rec = dict(card=card, sm_clock_after=smi("clocks.sm"), model="dagr-s + resnet50", width=W, height=H, streams=list(STREAMS),
           stream_rate_mev_s=RATE / 1e6, chunk_us=CHUNK, window_us=WINDOW, frame_us=FRAME, stream_seconds=SECONDS, runs=runs,
           since_frame_extra_device_us=extra,
           note="two rounds in one process, for each S the sliding and since_frame routes alternated (the order swapped in round 1); "
                "latency = host wall clock from submit() until the detections of all cameras are on the host, steps submitted back "
                "to back; device_ms = CUDA events around the step on the detector's stream; live_events_mean = live events per "
                "step and camera after the step; frame_to_first_use_ms = host time from set_frame until the detections of the "
                "first step using the frame are on the host, all cameras pooled; frames are never waited for; "
                "since_frame_extra_device_us = the D2D control-block copy + the second dagr_stream_push[_multi] alone, 200 per "
                "captured graph, per replay / 200; card = nvidia-smi name, power limit, max SM clock and SM clock at the start")
(out_dir / "h100_interframe_stream.json").write_text(json.dumps(rec, indent=1))
print("wrote", out_dir / "h100_interframe_stream.json")
