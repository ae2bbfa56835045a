"""Camera frames straight from the sensor (raw_frames=True) against preparing them on the host, in one process: dagr-s +
ResNet-50 at 320x215 on S raw 640x480 hybrid cameras (events as in tools/raw_stream_bench.py: 4 Mevents/s raw per camera,
uniform, 1 ms chunks, 50 ms window, sensor=(640, 480)), a new 640x480 frame every 50 ms of stream time per camera, camera s
offset by s * 50 / S ms; S in {1, 8}.  For each S, alternated in two rounds:
  raw    FusionMultiStreamDetector(sensor=(640, 480), raw_frames=True): set_frame takes the camera's u8 [480, 640, 3] frame;
         H2D of 922 KB, dagr_frame_preprocess (crop, cubic 2x down-sizing, HWC -> CHW, / 255) on the frame stream
  host   the same detector without raw_frames: the frame is cropped and resized on the host first (cv2.resize(INTER_CUBIC)
         where OpenCV is importable, else the integer restatement oracle/ref_frame.py; `host_resize` records which), then
         set_frame takes the u8 [3, 215, 320] frame (H2D of 206 KB, `.float() / 255.0`)
Per route: set_frame host time (host: including the resize), frame-to-first-use (host time from the frame's arrival to the
detections of the first step that used it), step latency.  Beside them: dagr_frame_preprocess device time on one frame and
on 8 frames (f32 and u8 outputs; CUDA events around a captured graph of back-to-back launches) and the host resize alone.
Writes OUT/h100_raw_frames.json (usage: python tools/raw_frame_bench.py OUT)."""
import gc
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200 import ingest
from dagr_b200.model.dagr import DAGR
from dagr_b200.streaming import FusionMultiStreamDetector, synth_stream
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

SW, SH, W, H, SCALE = 640, 480, 320, 215, 2
RATE, CHUNK, WINDOW, SECONDS, FRAME_US, MAX_CHUNK = 4_000_000, 1000, 50_000, 1.0, 50_000, 8192
STREAMS = (1, 8)
WARM = WINDOW // CHUNK + 20                                              # fill the window (+ capture) before timing

if len(sys.argv) != 2:
    sys.exit("usage: python tools/raw_frame_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")

try:
    import cv2
    HOST_RESIZE = f"cv2 {cv2.__version__} resize(INTER_CUBIC)"

    def host_prep(img):
        return torch.from_numpy(np.ascontiguousarray(cv2.resize(img[:SCALE * H], (W, H), interpolation=cv2.INTER_CUBIC).transpose(2, 0, 1)))
except ImportError:
    from oracle.ref_frame import preprocess_image
    HOST_RESIZE = "oracle/ref_frame.py preprocess_image (numpy, OpenCV not importable)"

    def host_prep(img):
        return torch.from_numpy(preprocess_image(img, H, W, SCALE)[0])


def card(q="name,power.limit,clocks.max.sm,clocks.sm"):
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


print("card (name, power limit, max SM clock, SM clock):", card(), "| host resize:", HOST_RESIZE, flush=True)
torch.manual_seed(0)
model = randomize_bn(DAGR(default_args("s", batch_size=1, use_image=True, img_net="resnet50"), height=H, width=W).eval()).to(dev)
total_s = SECONDS + WINDOW * 1e-6 + 0.02
grid = np.arange(0, int(total_s * 1e6) + CHUNK, CHUNK)
NCH = len(grid) - 1
cams = []
for s in range(max(STREAMS)):
    x, y, t, p = synth_stream(RATE, total_s, SW, SH, seed=99 + s, kind="uniform")
    cams.append((x.astype(np.uint16), y.astype(np.uint16), t.astype(np.int64), ((p + 1) // 2).astype(np.int8)))
bounds = [np.searchsorted(c[2], grid) for c in cams]
rng = np.random.default_rng(0)
frames = [rng.integers(0, 256, (SH, SW, 3), dtype=np.uint8) for _ in range(4)]
q = lambda v, f: v[min(len(v) - 1, int(f * len(v)))]


def dist(v):
    v = sorted(v)
    return dict(n=len(v), p50=q(v, 0.5), p99=q(v, 0.99), max=v[-1]) if v else dict(n=0)


def run(route, S):
    raw = route == "raw"
    det = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=MAX_CHUNK, sensor=(SW, SH), raw_frames=raw)
    offset = [(s * FRAME_US // S) // CHUNK * CHUNK for s in range(S)]
    set_ms, lat, dev_ms = [], [], []
    first_use = [[] for _ in range(S)]
    waiting = {}                                                         # (camera, frame id) -> host time the frame arrived
    for s in range(S):
        det.set_frame(s, frames[s % 4] if raw else host_prep(frames[s % 4]), t_us=0)
    gc_was = gc.isenabled()
    gc.collect()
    gc.disable()                                                         # a collector pause inside a 1 ms period is a latency spike
    for k in range(NCH):
        tk, timed = k * CHUNK, k >= WARM
        for s in range(S):
            if tk > offset[s] and (tk - offset[s]) % FRAME_US == 0:      # camera s delivers a frame at stream time tk
                img = frames[(s + (tk - offset[s]) // FRAME_US) % 4]
                ts = time.perf_counter()
                fid = det.set_frame(s, img if raw else host_prep(img), t_us=tk)
                if timed:
                    set_ms.append((time.perf_counter() - ts) * 1e3)
                    waiting[(s, fid)] = ts
        chunks = [tuple(v[int(bounds[s][k]):int(bounds[s][k + 1])] for v in cams[s]) for s in range(S)]
        t_end = [int(grid[k + 1])] * S
        if timed:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(det.stream)
        det.submit(chunks, t_end)
        if timed:
            e1.record(det.stream)
        det.result()
        if timed:
            t1 = time.perf_counter()
            lat.append((t1 - t0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            for s, cam in enumerate(det._cams):
                key = (s, cam.step_frame[0])
                if key in waiting:
                    first_use[s].append((t1 - waiting.pop(key)) * 1e3)
    if gc_was:
        gc.enable()
    torch.cuda.synchronize(dev)
    return dict(route=route, streams=S, steps=len(lat), frames=len(set_ms), set_frame_host_ms=dist(set_ms),
                frame_to_first_use_ms=dist([v for u in first_use for v in u]), latency_ms=dist(lat), device_ms=dist(dev_ms),
                overflow=[det.window_state(s)["overflow"] for s in range(S)])


def kernel_times():
    """dagr_frame_preprocess alone, per output kind and F: a CUDA graph of LAUNCHES back-to-back launches (so the device
    never waits for the host between them), replayed 40 times after 5 warm-up replays; CUDA events around each replay,
    divided by LAUNCHES."""
    LAUNCHES = 50
    lut = ingest.frame_lut(dev)
    res = {}
    side = torch.cuda.Stream(device=dev)
    for F in (1, 8):
        src = torch.from_numpy(np.stack([frames[i % 4] for i in range(F)])).to(dev)
        for kind in ("f32", "u8"):
            tab = lut if kind == "f32" else None
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                ingest.preprocess_frames(src, H, W, SCALE, tab)         # module load, outside the capture
            torch.cuda.synchronize(dev)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                for _ in range(LAUNCHES):
                    ingest.preprocess_frames(src, H, W, SCALE, tab)
            ts = []
            for i in range(45):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                e1.synchronize()
                if i >= 5:
                    ts.append(e0.elapsed_time(e1) * 1e3 / LAUNCHES)
            res[f"F{F}_{kind}_us"] = dist(ts)
            del g
    ts = []
    for i in range(220):
        t0 = time.perf_counter()
        host_prep(frames[i % 4])
        if i >= 20:
            ts.append((time.perf_counter() - t0) * 1e3)
    res["host_resize_ms"] = dist(ts)
    return res


runs = []
for rnd in range(2):
    kt = kernel_times()
    kt["round"] = rnd
    print(f"round {rnd} kernel: " + ", ".join(f"{k} p50 {v['p50']:.2f}" for k, v in kt.items() if k != "round"), flush=True)
    runs.append(dict(kind="kernel", **kt))
    for S in STREAMS:
        for route in ("raw", "host"):
            t0 = time.time()
            r = run(route, S)
            r["round"] = rnd
            runs.append(r)
            print(f"round {rnd} S={S} {route:4s}: set_frame p50 {r['set_frame_host_ms']['p50']:.3f} max {r['set_frame_host_ms']['max']:.3f} ms, "
                  f"first use p50 {r['frame_to_first_use_ms']['p50']:.2f} max {r['frame_to_first_use_ms']['max']:.2f} ms, step p50 "
                  f"{r['latency_ms']['p50']:.3f} p99 {r['latency_ms']['p99']:.3f} ms, frames {r['frames']} ({time.time() - t0:.0f} s)",
                  flush=True)

rec = dict(card=card(), sm_clock_after=card("clocks.sm"), model="dagr-s + resnet50", width=W, height=H, sensor=[SW, SH],
           raw_rate_mev_s_per_camera=RATE / 1e6, chunk_us=CHUNK, window_us=WINDOW, frame_us=FRAME_US, stream_seconds=SECONDS,
           streams=list(STREAMS), host_resize=HOST_RESIZE, runs=runs,
           note="card = nvidia-smi name, power limit, max SM clock and SM clock at the start; set_frame_host_ms = host time of "
                "set_frame, for the host route including the host resize; frame_to_first_use_ms = host time from a frame's arrival "
                "until the detections of the first step using it are on the host (all cameras pooled); latency_ms = submit() until "
                "the detections of all cameras are on the host, steps back to back; device_ms = CUDA events around submit() on the "
                "detector's stream; kernel F*_us = device time of one dagr_frame_preprocess launch on F device-resident 640x480 "
                "frames (CUDA events around a graph replay of 50 back-to-back launches, divided by 50); Python's cyclic garbage collector is paused during the timed loops")
(out_dir / "h100_raw_frames.json").write_text(json.dumps(rec, indent=1))
print("wrote", out_dir / "h100_raw_frames.json")
