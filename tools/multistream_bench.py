"""S event cameras on one GPU (MultiStreamDetector) against the single-stream detector, in one process:
dagr-l, 640x480, 1 Mevents/s per stream in 1 ms chunks, 50 ms live window, 2 s of stream; S in {1, 2, 4, 8} on the uniform
stream and S = 8 on the clustered one, each run preceded by a run of the single-stream stream_benchmark (the config-5
bench key) so that both see the same clocks.  Then a torch.profiler trace of 30 replayed S = 8 steps for the H2D copy of
the packed stage.  Writes OUT/h100_multistream.json (usage: python tools/multistream_bench.py OUT)."""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200.model.dagr import DAGR
from dagr_b200.streaming import MultiStreamDetector, multistream_benchmark, stream_benchmark, synth_stream
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

W, H = 640, 480
if len(sys.argv) != 2:
    sys.exit("usage: python tools/multistream_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
torch.manual_seed(0)
model = randomize_bn(DAGR(default_args("l", batch_size=1), height=H, width=W).eval()).to(dev)

runs = []
for S, kind in ((1, "uniform"), (2, "uniform"), (4, "uniform"), (8, "uniform"), (8, "clustered")):
    t0 = time.time()
    single = stream_benchmark(dev, size="l", width=W, height=H, kind=kind, model=model)
    multi = multistream_benchmark(dev, S, size="l", width=W, height=H, kind=kind, model=model)
    runs.append(dict(streams=S, kind=kind, single=single, multi=multi))
    print(f"S={S} {kind}: single p50 {single['latency_ms']['p50']:.3f} ms | multi p50 {multi['latency_ms']['p50']:.3f} p99 "
          f"{multi['latency_ms']['p99']:.3f} ms, device {multi['device_ms']['p50']:.3f} ms, {multi['sustained_mev_s']:.2f} Mev/s, "
          f"live {multi['live_events']}, overflow {multi['overflow']} ({time.time() - t0:.0f} s)", flush=True)

# H2D of the packed stage (fixed size S*max_chunk*16 bytes) in a trace of replayed S = 8 steps
S, chunk_us = 8, 1000
evs = [synth_stream(1_000_000, 0.12, W, H, seed=99 + s) for s in range(S)]
det = MultiStreamDetector(model, streams=S, window_us=50_000, max_chunk=4096)
grid = np.arange(0, 120_001, chunk_us)
bounds = [np.searchsorted(e[2], grid) for e in evs]


def step(k):
    det.push([(e[0][b[k]:b[k + 1]], e[1][b[k]:b[k + 1]], e[2][b[k]:b[k + 1]], e[3][b[k]:b[k + 1]]) for e, b in zip(evs, bounds)],
             [(k + 1) * chunk_us] * S)


for k in range(80):
    step(k)
from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for k in range(80, 110):
        step(k)
h2d = [e.device_time_total for e in prof.events() if "HtoD" in e.name]
stage = dict(stage_bytes=det.stage_bytes, h2d_copies=len(h2d),
             h2d_us_mean=(float(np.mean(h2d)) if h2d else None), h2d_us_max=(float(np.max(h2d)) if h2d else None),
             note="torch.profiler, 30 replayed S = 8 steps (1 Mevents/s per stream, max_chunk 4096): device time of the "
                  "host-to-device copies in the trace (the packed stage is the only H2D copy of a step)")
print("stage H2D:", stage, flush=True)

rec = dict(card=card, model="dagr-l", width=W, height=H, stream_rate_mev_s_per_stream=1.0, chunk_us=1000, window_us=50_000,
           stream_seconds=2.0, runs=runs, stage_h2d=stage,
           note="each multi-stream run follows a single-stream run (stream_benchmark, the config-5 bench key) on the same "
                "model in the same process; latency = host submit until the detections of all S streams are on the host")
(out_dir / "h100_multistream.json").write_text(json.dumps(rec, indent=1))
print("wrote", out_dir / "h100_multistream.json")
