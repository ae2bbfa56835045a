"""The bf16 image branch (DAGR.image_precision = "bf16") against the default TF32 one, in one process, alternating the two
precisions in each of two rounds, on config 3's model (dagr-s + ResNet-50, 640x480, random weights with randomised BN):
  * config 3: the synchronous forward on ten growing windows (linspace(0, 50 ms, 10) of a 300 k events/sample uniform
    window, as bench.py's interframe_latency_ms), B = 8 and B = 1: ms per forward (CUDA events, mean of 3 after 2 warm-ups);
  * the trunk's device time per frame (CUDA events around the branch on FusionStreamingDetector's frame stream);
  * FusionStreamingDetector on config 5's stream (1 Mevents/s in 1 ms chunks, 50 ms window) with a frame every 50 ms: chunk
    p50 / p99, the p50 of the chunks that overlap a trunk, frame to first use p50 / max;
  * FusionMultiStreamDetector at S = 8 (1 Mevents/s per camera, a frame every 50 ms per camera): step p50, frame to first use;
  * the precision cost on seeded inputs (tests/test_bf16_image_gpu.py:bf16_precision_report).
Then, in a separate profiled run, the device time of the three image-sampling kernels in both formats (torch.profiler).
The card's name, power limit and SM clocks are read in the same call.  Writes OUT/h100_bf16_image.json
(usage: python tools/bf16_image_bench.py OUT)."""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200.data import EventBatch, format_data, synth_batch
from dagr_b200.model.dagr import DAGR
from dagr_b200.streaming import fusion_multistream_benchmark, fusion_stream_benchmark
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

W, H, T = 640, 480, 1_000_000
PRECISIONS = ("tf32", "bf16")
if len(sys.argv) != 2:
    sys.exit("usage: python tools/bf16_image_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")
smi = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"]
card = subprocess.run(smi, capture_output=True, text=True).stdout.strip()
print("card (name, power limit, max SM clock, SM clock):", card, flush=True)


def model_s(B):
    torch.manual_seed(0)
    return randomize_bn(DAGR(default_args("s", batch_size=B, use_image=True, img_net="resnet50"), height=H, width=W).eval()).to(dev)


def windows(B):
    d = format_data(synth_batch(B, 300_000, W, H, seed=4242, kind="uniform", with_image=True).to(dev))
    t_us = (d.pos[:, 2].double() * T).round()
    subs = []
    for n_us in np.linspace(0, 50000, 10):
        msk = t_us < (T - 50000 + n_us)
        subs.append(EventBatch(x=d.x[msk], pos=d.pos[msk], batch=d.batch[msk], width=d.width, height=d.height,
                               time_window=d.time_window, image=d.image, num_graphs=B, dims=(W, H, T)))
    return subs


def interframe(m, subs):
    ms = []
    for sub in subs:
        for _ in range(2):
            m(sub.clone())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            m(sub.clone())
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / 3)
    return dict(ms=[round(v, 4) for v in ms], p50_ms=float(np.median(ms)), max_ms=max(ms))


def short(r):
    keep = ("latency_ms", "latency_ms_trunk_in_flight", "device_ms", "trunk_device_ms", "frame_to_first_use_ms", "sustained_mev_s",
            "steps_trunk_in_flight")
    return {k: r[k] for k in keep if k in r}


models = {B: model_s(B) for B in (8, 1)}
subs = {B: windows(B) for B in (8, 1)}
runs = []
for rnd in range(2):
    t0 = time.time()
    rec = dict(round=rnd)
    for prec in PRECISIONS:
        r = {}
        for B in (8, 1):
            models[B].image_precision = prec
            r[f"config3_batch{B}"] = interframe(models[B], subs[B])
            print(f"round {rnd} {prec} config 3 B={B}: p50 {r[f'config3_batch{B}']['p50_ms']:.3f} ms, max "
                  f"{r[f'config3_batch{B}']['max_ms']:.3f} ms", flush=True)
        m1 = models[1]
        r["fusion_stream"] = short(fusion_stream_benchmark(dev, model=m1))
        fs = r["fusion_stream"]
        print(f"round {rnd} {prec} fusion stream: chunk p50 {fs['latency_ms']['p50']:.3f} p99 {fs['latency_ms']['p99']:.3f}, "
              f"trunk in flight p50 {fs['latency_ms_trunk_in_flight'].get('p50', float('nan')):.3f}, trunk "
              f"{fs['trunk_device_ms']['p50']:.3f} ms, first use p50 {fs['frame_to_first_use_ms']['p50']:.3f} max "
              f"{fs['frame_to_first_use_ms']['max']:.3f} ms", flush=True)
        r["fusion_multistream_s8"] = short(fusion_multistream_benchmark(dev, 8, model=m1))
        ms = r["fusion_multistream_s8"]
        print(f"round {rnd} {prec} S=8: step p50 {ms['latency_ms']['p50']:.3f} p99 {ms['latency_ms']['p99']:.3f} ms, trunk "
              f"{ms['trunk_device_ms']['p50']:.3f} ms, first use p50 {np.median([v['p50'] for v in ms['frame_to_first_use_ms']]):.3f} ms",
              flush=True)
        rec[prec] = r
    runs.append(rec)
    print(f"round {rnd}: {time.time() - t0:.0f} s", flush=True)
card_after = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

# precision cost on seeded inputs
from tests.test_bf16_image_gpu import bf16_precision_report
precision = [bf16_precision_report(B=2, seed=s) for s in (0, 1)]
print("precision:", precision, flush=True)

# device time of the image-sampling kernels in both formats: one profiled config-3 forward per precision at B = 8
from torch.profiler import ProfilerActivity, profile
kernels = {}
m8 = models[8]
for prec in PRECISIONS:
    m8.image_precision = prec
    m8(subs[8][-1].clone())
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            m8(subs[8][-1].clone())
        torch.cuda.synchronize()
    agg = {}
    for e in prof.events():
        for k in ("k_l1_x0_image", "k_voxel_sample_max", "k_sample_features"):
            if e.device_type == torch.autograd.DeviceType.CUDA and k in e.name:
                a = agg.setdefault(k, [0.0, 0])
                a[0] += e.device_time_total / 1e3
                a[1] += 1
    kernels[prec] = {k: dict(ms_per_forward=v[0] / 5, launches_per_forward=v[1] / 5) for k, v in agg.items()}
    print(f"kernels {prec}:", kernels[prec], flush=True)

rec = dict(card=card, sm_clock_after=card_after, model="dagr-s + resnet50", width=W, height=H, runs=runs, precision=precision,
           kernels_b8_full_window=kernels,
           note="two rounds in one process, tf32 then bf16 in each; config 3 = synchronous forward on 10 growing windows of a "
                "300 k events/sample uniform window (mean of 3 after 2 warm-ups each); fusion_stream = fusion_stream_benchmark "
                "(1 Mevents/s, 1 ms chunks, 50 ms window, a frame every 50 ms); fusion_multistream_s8 = "
                "fusion_multistream_benchmark(streams=8); kernels = torch.profiler device time per B = 8 full-window forward; "
                "precision = bf16_precision_report on seeded B = 2 inputs (seeds 0, 1); card = nvidia-smi name, power limit, max "
                "SM clock and SM clock at the start")
(out_dir / "h100_bf16_image.json").write_text(json.dumps(rec, indent=1))
print("wrote", out_dir / "h100_bf16_image.json")
