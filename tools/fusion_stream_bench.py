"""Hybrid (image + events) streaming with FusionStreamingDetector against the events-only StreamingDetector, in one process:
config 3's model (dagr-s + ResNet-50, 640x480) on config 5's stream (1 Mevents/s in 1 ms chunks, 50 ms live window, 2 s of
stream) with a new camera frame every 50 ms of stream time (20 Hz).  Two rounds, each: the events-only stream_benchmark of
dagr-s (the cost of fusion per chunk is the difference), the fusion loop that never waits for a frame, the same loop with
sync_frame() after every set_frame, and the non-waiting loop with the steps on a higher-priority stream than the trunk.
Writes OUT/h100_fusion_stream.json (usage: python tools/fusion_stream_bench.py OUT)."""
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200.model.dagr import DAGR
from dagr_b200.streaming import fusion_stream_benchmark, stream_benchmark
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

W, H = 640, 480
if len(sys.argv) != 2:
    sys.exit("usage: python tools/fusion_stream_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card (name, power limit, max SM clock, SM clock):", card, flush=True)
torch.manual_seed(0)
fusion = randomize_bn(DAGR(default_args("s", batch_size=1, use_image=True, img_net="resnet50"), height=H, width=W).eval()).to(dev)
torch.manual_seed(0)
events_only = randomize_bn(DAGR(default_args("s", batch_size=1), height=H, width=W).eval()).to(dev)


def show(name, r):
    lat, tif = r["latency_ms"], r.get("latency_ms_trunk_in_flight", {})
    extra = ""
    if "trunk_device_ms" in r:
        extra = (f" | trunk in flight: n {tif['n']} p50 {tif.get('p50', float('nan')):.3f} p99 {tif.get('p99', float('nan')):.3f}"
                 f" | trunk {r['trunk_device_ms']['p50']:.3f} ms | first use p50 {r['frame_to_first_use_ms']['p50']:.3f}"
                 f" max {r['frame_to_first_use_ms']['max']:.3f} ms")
    print(f"{name}: p50 {lat['p50']:.3f} p99 {lat['p99']:.3f} max {lat['max']:.3f} ms, device p50 {r['device_ms']['p50']:.3f} ms"
          + extra, flush=True)


runs = []
for rnd in range(2):
    t0 = time.time()
    rec = dict(round=rnd)
    rec["events_only"] = stream_benchmark(dev, size="s", width=W, height=H, model=events_only)
    show("events-only dagr-s", rec["events_only"])
    rec["fusion"] = fusion_stream_benchmark(dev, model=fusion)
    show("fusion", rec["fusion"])
    rec["fusion_sync_frame"] = fusion_stream_benchmark(dev, model=fusion, sync_frames=True)
    show("fusion + sync_frame", rec["fusion_sync_frame"])
    rec["fusion_step_priority_high"] = fusion_stream_benchmark(dev, model=fusion, step_priority=-1)
    show("fusion, high-priority steps", rec["fusion_step_priority_high"])
    runs.append(rec)
    print(f"round {rnd}: {time.time() - t0:.0f} s", flush=True)

card_after = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
rec = dict(card=card, sm_clock_after=card_after, model="dagr-s + resnet50", width=W, height=H, stream_rate_mev_s=1.0, chunk_us=1000,
           window_us=50_000, frame_us=50_000, stream_seconds=2.0, runs=runs,
           note="two rounds in one process; each round runs the events-only dagr-s stream_benchmark, then the fusion loop without "
                "waiting for frames, with sync_frame() after every set_frame, and without waiting but with the steps on a "
                "priority -1 stream; card = nvidia-smi name, power limit, max SM clock and SM clock at the start")
(out_dir / "h100_fusion_stream.json").write_text(json.dumps(rec, indent=1))
print("wrote", out_dir / "h100_fusion_stream.json")
