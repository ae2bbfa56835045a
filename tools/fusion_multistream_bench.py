"""S hybrid (image + events) cameras on one GPU with FusionMultiStreamDetector, against the events-only MultiStreamDetector at
the same S and the single hybrid camera of FusionStreamingDetector, in one process: config 3's model (dagr-s + ResNet-50,
640x480) on S = 1, 2, 4, 8 copies of config 5's stream (1 Mevents/s per camera in 1 ms chunks, 50 ms live window, 2 s of
stream), a new frame every 50 ms of stream time per camera, camera s's frames offset by s * 50 / S ms.  Two rounds.
Writes OUT/h100_fusion_multistream.json (usage: python tools/fusion_multistream_bench.py OUT)."""
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200.model.dagr import DAGR
from dagr_b200.streaming import fusion_multistream_benchmark, fusion_stream_benchmark, multistream_benchmark
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

W, H = 640, 480
STREAMS = (1, 2, 4, 8)
if len(sys.argv) != 2:
    sys.exit("usage: python tools/fusion_multistream_bench.py OUT_DIR")
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
    lat, dv = r["latency_ms"], r["device_ms"]
    extra = ""
    if "trunk_device_ms" in r:
        fu = r["frame_to_first_use_ms"]
        fu = fu if isinstance(fu, list) else [fu]
        extra = (f" | trunk {r['trunk_device_ms'].get('p50', float('nan')):.3f} ms x {r['trunk_device_ms']['n']}"
                 f" | steps with a trunk in flight {r.get('steps_trunk_in_flight', r['latency_ms_trunk_in_flight']['n'])}"
                 f" | first use p50 per camera " + " ".join(f"{x.get('p50', float('nan')):.2f}" for x in fu))
    print(f"{name}: p50 {lat['p50']:.3f} p99 {lat['p99']:.3f} ms, device p50 {dv['p50']:.3f} p99 {dv['p99']:.3f} ms" + extra, flush=True)


runs = []
for rnd in range(2):
    t0 = time.time()
    rec = dict(round=rnd, fusion_multistream={}, events_only_multistream={})
    rec["fusion_single"] = fusion_stream_benchmark(dev, model=fusion)
    show("FusionStreamingDetector (S = 1)", rec["fusion_single"])
    for S in STREAMS:
        r = fusion_multistream_benchmark(dev, S, model=fusion)
        rec["fusion_multistream"][str(S)] = r
        show(f"FusionMultiStreamDetector S = {S}", r)
        r = multistream_benchmark(dev, S, size="s", model=events_only)
        rec["events_only_multistream"][str(S)] = r
        show(f"MultiStreamDetector events-only S = {S}", r)
    runs.append(rec)
    print(f"round {rnd}: {time.time() - t0:.0f} s", flush=True)

card_after = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
rec = dict(card=card, sm_clock_after=card_after, model="dagr-s + resnet50", width=W, height=H, streams=list(STREAMS),
           stream_rate_mev_s=1.0, chunk_us=1000, window_us=50_000, frame_us=50_000, stream_seconds=2.0, runs=runs,
           note="two rounds in one process; each round runs FusionStreamingDetector (one hybrid camera), then for every S the "
                "FusionMultiStreamDetector loop (frames never waited for) and the events-only dagr-s MultiStreamDetector loop; "
                "card = nvidia-smi name, power limit, max SM clock and SM clock at the start")
(out_dir / "h100_fusion_multistream.json").write_text(json.dumps(rec, indent=1))
print("wrote", out_dir / "h100_fusion_multistream.json")
