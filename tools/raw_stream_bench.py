"""Raw sensor streaming (sensor=(640, 480)) against the routes a DSEC camera has without it, in one process: dagr-l at
320x215 on S raw 640x480 cameras at 4 Mevents/s each (uniform positions and polarities, seeds 99, 100, ...) in 1 ms chunks,
50 ms live window, S in {1, 2, 4, 8}.  For each S, alternated in two rounds:
  raw        MultiStreamDetector(sensor=(640, 480)) fed the raw chunks: H2D of the raw stage, dagr_stream_ingest, push, forward
  host       the same detector without a sensor fed chunks down-sampled, cropped and rebased before the timed loop (the
             lower bound: what the model costs when the ingest is free)
  roundtrip  what users have without this mode: per camera and chunk, H2D of the raw chunk, ingest.downsample_events (one
             host sync), D2H, crop and rebase in numpy, then submit to the detector without a sensor
plus the device time of dagr_stream_ingest alone (CUDA events around eager launches on the raw stages of the timed steps).
Writes OUT/h100_raw_stream.json (usage: python tools/raw_stream_bench.py OUT)."""
import gc
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200 import _lib, ingest
from dagr_b200.model.dagr import DAGR
from dagr_b200.streaming import MultiStreamDetector, synth_stream
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

SW, SH, W, H = 640, 480, 320, 215
RATE, CHUNK, WINDOW, SECONDS, MAX_CHUNK = 4_000_000, 1000, 50_000, 1.0, 8192
WARM = WINDOW // CHUNK + 20                                              # fill the window (+ capture) before timing

if len(sys.argv) != 2:
    sys.exit("usage: python tools/raw_stream_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


print("card:", card(), flush=True)
torch.manual_seed(0)
model = randomize_bn(DAGR(default_args("l", batch_size=1), height=H, width=W).eval()).to(dev)
total_s = SECONDS + WINDOW * 1e-6 + 0.02
grid = np.arange(0, int(total_s * 1e6) + CHUNK, CHUNK)
NCH = len(grid) - 1
cams = []
for s in range(8):
    x, y, t, p = synth_stream(RATE, total_s, SW, SH, seed=99 + s, kind="uniform")
    cams.append((x.astype(np.uint16), y.astype(np.uint16), t.astype(np.int64), ((p + 1) // 2).astype(np.int8)))
bounds = [np.searchsorted(c[2], grid) for c in cams]


def raw_chunk(s, k):
    a, b = int(bounds[s][k]), int(bounds[s][k + 1])
    return tuple(v[a:b] for v in cams[s])


def predownsample(s):
    """camera s's chunks as the detector without a sensor takes them: ingest.downsample_events on the GPU with the change
    map carried, crop y < H, t rebased to the first raw timestamp, polarity 2p - 1."""
    cm, base, out = None, int(cams[s][2][0]), []
    for k in range(NCH):
        x, y, t, p = raw_chunk(s, k)
        ev = dict(x=torch.from_numpy(x.astype(np.int16)).to(dev), y=torch.from_numpy(y.astype(np.int16)).to(dev),
                  t=torch.from_numpy(t).to(dev), p=torch.from_numpy(2 * p - 1).to(dev))
        o, cm = ingest.downsample_events(ev, SH, SW, SH // 2, SW // 2, change_map=cm)
        o = {q: v.cpu().numpy() for q, v in o.items()}
        keep = o["y"] < H
        out.append((o["x"][keep], o["y"][keep], (o["t"][keep] - base).astype(np.int32), o["p"][keep]))
    return out


pre = [predownsample(s) for s in range(8)]
q = lambda v, f: v[min(len(v) - 1, int(f * len(v)))]


def dist(v):
    v = sorted(v)
    return dict(p50=q(v, 0.5), p99=q(v, 0.99), max=v[-1])


def run(route, S):
    raw = route == "raw"
    det = MultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=MAX_CHUNK, sensor=(SW, SH) if raw else None)
    bases = [int(cams[s][2][0]) for s in range(S)]
    lat, dev_ms, nraw, nkept = [], [], [], []
    stages = []
    gc_was = gc.isenabled()
    gc.collect()
    gc.disable()                                                         # a collector pause inside a 1 ms period is a latency spike
    cms = [None] * S                                                     # roundtrip: the change maps it carries
    for k in range(NCH):
        timed = k >= WARM
        t0 = time.perf_counter()
        if raw:
            chunks, t_end = [raw_chunk(s, k) for s in range(S)], [int(grid[k + 1])] * S
        elif route == "host":
            chunks, t_end = [pre[s][k] for s in range(S)], [int(grid[k + 1]) - bases[s] for s in range(S)]
        else:
            chunks = []
            for s in range(S):
                x, y, t, p = raw_chunk(s, k)
                ev = dict(x=torch.from_numpy(x.astype(np.int16)).to(dev), y=torch.from_numpy(y.astype(np.int16)).to(dev),
                          t=torch.from_numpy(t).to(dev), p=torch.from_numpy(2 * p - 1).to(dev))
                o, cms[s] = ingest.downsample_events(ev, SH, SW, SH // 2, SW // 2, change_map=cms[s])
                o = {q_: v.cpu().numpy() for q_, v in o.items()}
                keep = o["y"] < H
                chunks.append((o["x"][keep], o["y"][keep], (o["t"][keep] - bases[s]).astype(np.int32), o["p"][keep]))
            t_end = [int(grid[k + 1]) - bases[s] for s in range(S)]
        if timed:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(det.stream)
        det.submit(chunks, t_end)
        if timed:
            e1.record(det.stream)
        det.result()
        if timed:
            lat.append((time.perf_counter() - t0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            st = [det.window_state(s) for s in range(S)]
            nkept.append(sum(x["appended"] for x in st))
            nraw.append(sum(len(raw_chunk(s, k)[2]) for s in range(S)))
            if raw and len(stages) < 200:
                stages.append(det.stage_h.clone())
    if gc_was:
        gc.enable()
    res = dict(route=route, streams=S, steps=len(lat), latency_ms=dist(lat), device_ms=dist(dev_ms),
               raw_mev_s_per_camera=float(np.sum(nraw)) / len(lat) / S / CHUNK, kept_mev_s_per_camera=float(np.sum(nkept)) / len(lat) / S / CHUNK,
               kept_fraction=float(np.sum(nkept)) / float(np.sum(nraw)), live_events=[det.window_state(s)["live"] for s in range(S)],
               overflow=[det.window_state(s)["overflow"] for s in range(S)])
    if raw:                                                              # dagr_stream_ingest alone on the raw stages of the timed steps
        lib = _lib.load()
        cm = det._cmap.clone()
        rd = torch.empty_like(det.raw_d)
        out = torch.empty_like(det.stage_d)
        ts = []
        for i, sh in enumerate(stages):
            rd.copy_(sh)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(lib.dagr_stream_ingest(_lib.ptr(rd), S, MAX_CHUNK, 2, 2, SW // 2, SH // 2, H, _lib.ptr(cm), _lib.ptr(out), MAX_CHUNK,
                                              _lib.stream_ptr()), "stream_ingest")
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        res["ingest_kernel_us"] = dist(ts)
        res["ingest_share_of_step_p50"] = res["ingest_kernel_us"]["p50"] * 1e-3 / res["device_ms"]["p50"]
    return res


runs = []
for rnd in range(2):
    for S in (1, 2, 4, 8):
        for route in ("raw", "host", "roundtrip"):
            t0 = time.time()
            r = run(route, S)
            r["round"] = rnd
            runs.append(r)
            extra = f", ingest {r['ingest_kernel_us']['p50']:.1f} us ({100 * r['ingest_share_of_step_p50']:.1f} %)" if route == "raw" else ""
            print(f"round {rnd} S={S} {route:9s}: p50 {r['latency_ms']['p50']:.3f} p99 {r['latency_ms']['p99']:.3f} ms, device "
                  f"{r['device_ms']['p50']:.3f} ms, raw {r['raw_mev_s_per_camera']:.2f} kept {r['kept_mev_s_per_camera']:.3f} Mev/s "
                  f"per camera{extra}, overflow {r['overflow']} ({time.time() - t0:.0f} s)", flush=True)

rec = dict(card=card(), model="dagr-l", width=W, height=H, sensor=[SW, SH], raw_rate_mev_s_per_camera=RATE / 1e6, chunk_us=CHUNK,
           window_us=WINDOW, stream_seconds=SECONDS, max_chunk=MAX_CHUNK, runs=runs,
           note="latency = host wall clock from submit() until the detections of all cameras are on the host, steps back to back; "
                "device_ms = CUDA events around submit() on the detector's stream (for roundtrip the per-camera down-sampling "
                "before it is in the host latency only); ingest_kernel_us = CUDA events around eager "
                "dagr_stream_ingest launches on the raw stages of the first 200 timed steps; kept = events appended to the rings "
                "(down-sampled 2x2 and cropped to 215 rows); Python's cyclic garbage collector is paused during the timed loops")
(out_dir / "h100_raw_stream.json").write_text(json.dumps(rec, indent=1))
print("wrote", out_dir / "h100_raw_stream.json")
