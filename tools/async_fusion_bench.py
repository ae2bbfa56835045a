"""Incremental updates of the hybrid (image + events) model with AsyncDAGR: config 3's model (dagr-s + ResNet-50, 640x480,
B = 1) initialised on a 50 ms window of a 1 Mevents/s stream, then UPDATES updates of 1000 events each (append-only, one
frame).  Reports, in one process:
  * the update's device time (CUDA events around the step, the host waits for every step) and host latency, p50 / p99,
    plus the first and last 50 updates (the live count grows by 1000 events per update);
  * the per-op split of an update from engine.prof (a separate profiled run), x0 resampling and voxel_sample_max_inc among
    them, and x0's share of the summed op time;
  * the cost of a frame-change rebuild (a step with a new frame: trunk + one full pass over every event seen so far);
  * the dense model(data) forward over the same events (at the first update's count and at the last one's);
  * the events-only dagr-s AsyncDAGR update on the same events.
Writes OUT/h100_async_fusion.json (usage: python tools/async_fusion_bench.py OUT [UPDATES])."""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200.asynchronous import AsyncDAGR
from dagr_b200.data import EventBatch
from dagr_b200.model.dagr import DAGR
from dagr_b200.streaming import synth_stream
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

W, H, INIT_US, CHUNK = 640, 480, 50_000, 1000
if len(sys.argv) not in (2, 3):
    sys.exit("usage: python tools/async_fusion_bench.py OUT_DIR [UPDATES]")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
UPDATES = int(sys.argv[2]) if len(sys.argv) == 3 else 500
dev = torch.device("cuda:0")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card (name, power limit, max SM clock, SM clock):", card, flush=True)
torch.manual_seed(0)
fusion = randomize_bn(DAGR(default_args("s", batch_size=1, use_image=True, img_net="resnet50"), height=H, width=W).eval()).to(dev)
torch.manual_seed(0)
events_only = randomize_bn(DAGR(default_args("s", batch_size=1), height=H, width=W).eval()).to(dev)

x, y, t, p = synth_stream(1_000_000, (INIT_US + (UPDATES + 10) * CHUNK) * 1e-6, W, H, seed=99)
pos_all = torch.from_numpy(np.stack([x, y, t], 1).astype(np.int32)).to(dev)
pol_all = torch.from_numpy(p.astype(np.float32)).to(dev)
N0 = int(np.searchsorted(t, INIT_US))
g = torch.Generator().manual_seed(3)
frames = [(torch.randint(0, 256, (1, 3, H, W), generator=g, dtype=torch.uint8).float() / 255.0).to(dev) for _ in range(2)]


def chunk(a, b, image=None):
    """events [a, b) of the stream as a formatted batch (denormalised positions, as the streaming front end hands them over)."""
    n = b - a
    return EventBatch(x=pol_all[a:b].view(-1, 1), pos=torch.zeros(n, 3, device=dev), batch=torch.zeros(n, dtype=torch.long, device=dev),
                      width=torch.tensor([W]), height=torch.tensor([H]), time_window=torch.tensor([1_000_000]), pos_denorm=pos_all[a:b],
                      num_graphs=1, dims=(W, H, 1_000_000), image=image)


def stats(v):
    v = np.asarray(v, dtype=np.float64)
    return dict(n=int(v.size), p50=float(np.percentile(v, 50)), p99=float(np.percentile(v, 99)), mean=float(v.mean()), max=float(v.max()))


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    h0 = time.perf_counter()
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return out, e0.elapsed_time(e1), (time.perf_counter() - h0) * 1e3


def updates(model, n_updates, image):
    """init on the first INIT_US of the stream, then n_updates steps of CHUNK events -> (wrapper, device ms, host ms)."""
    a = AsyncDAGR(model)
    a.step_decoded(chunk(0, N0, image), batch_size=1)
    torch.cuda.synchronize()
    dms, hms = [], []
    for k in range(n_updates):
        _, d, h = timed(lambda: a.step_decoded(chunk(N0 + k * CHUNK, N0 + (k + 1) * CHUNK), batch_size=1))
        dms.append(d)
        hms.append(h)
    return a, dms, hms


def update_record(dms, hms, a):
    return dict(device_ms=stats(dms), host_ms=stats(hms), device_ms_first50=stats(dms[:50]), device_ms_last50=stats(dms[-50:]),
                live_events_first=N0 + CHUNK, live_events_last=a.num_events)


rec = dict(card=card, model="dagr-s + resnet50", width=W, height=H, batch=1, stream_rate_mev_s=1.0, init_window_us=INIT_US,
           init_events=N0, update_events=CHUNK, updates=UPDATES)
t_start = time.time()
updates(fusion, 50, frames[0])                                       # warm-up: kernels, branch graphs, workspaces
updates(events_only, 50, None)

a, dms, hms = updates(fusion, UPDATES, frames[0])
rec["fusion_update"] = update_record(dms, hms, a)
print(f"fusion update: device p50 {rec['fusion_update']['device_ms']['p50']:.3f} p99 {rec['fusion_update']['device_ms']['p99']:.3f} ms, "
      f"first 50 p50 {rec['fusion_update']['device_ms_first50']['p50']:.3f}, last 50 p50 {rec['fusion_update']['device_ms_last50']['p50']:.3f} "
      f"(live {N0 + CHUNK} .. {a.num_events})", flush=True)

# frame change: a step with a new frame re-seeds the state with one full pass over every event seen so far
n = a.num_events
rebuild = []
for k in range(6):
    _, d, _ = timed(lambda: a.step_decoded(chunk(n + k * CHUNK, n + (k + 1) * CHUNK, frames[(k + 1) % 2].clone()), batch_size=1))
    rebuild.append(d)
rec["frame_change_rebuild"] = dict(device_ms=stats(rebuild), live_events=a.num_events, frames=a.frames)
print(f"frame-change rebuild: device p50 {rec['frame_change_rebuild']['device_ms']['p50']:.3f} ms over {a.num_events} events", flush=True)
n_last = N0 + UPDATES * CHUNK
del a

# dense synchronous forward over the same events
rec["dense_forward"] = {}
for name, nev in (("first_update", N0 + CHUNK), ("last_update", n_last)):
    data = chunk(0, nev, frames[0])
    for _ in range(3):
        fusion.forward_decoded(data)
    dd = [timed(lambda: fusion.forward_decoded(data))[1] for _ in range(20)]
    rec["dense_forward"][name] = dict(events=nev, device_ms=stats(dd))
    print(f"dense model(data) over {nev} events: device p50 {rec['dense_forward'][name]['device_ms']['p50']:.3f} ms", flush=True)

# events-only dagr-s, same updates
a, dms, hms = updates(events_only, UPDATES, None)
rec["events_only_update"] = update_record(dms, hms, a)
print(f"events-only update: device p50 {rec['events_only_update']['device_ms']['p50']:.3f} p99 "
      f"{rec['events_only_update']['device_ms']['p99']:.3f} ms", flush=True)
del a

# per-op split of the fusion update (profiled run of its own: per-op events, eager coarse stack)
a = AsyncDAGR(fusion)
a.step_decoded(chunk(0, N0, frames[0]), batch_size=1)
torch.cuda.synchronize()
fusion.engine.prof = {}
NP = min(UPDATES, 100)
for k in range(NP):
    a.step_decoded(chunk(N0 + k * CHUNK, N0 + (k + 1) * CHUNK), batch_size=1)
torch.cuda.synchronize()
ops = fusion.engine.prof_summary()
fusion.engine.prof = None
total = sum(v["ms"] * v["calls"] for v in ops.values()) / NP
rec["fusion_update_ops"] = dict(updates=NP, live_events_last=a.num_events, ops_ms_per_update={k: v["ms"] * v["calls"] / NP for k, v in ops.items()},
                                sum_ms_per_update=total,
                                x0_share_of_op_time=(ops["l1_x0_image"]["ms"] * ops["l1_x0_image"]["calls"] / NP) / total)
for k, v in sorted(rec["fusion_update_ops"]["ops_ms_per_update"].items(), key=lambda kv: -kv[1])[:12]:
    print(f"  {k}: {v:.4f} ms per update", flush=True)
print(f"x0 share of the summed op time: {rec['fusion_update_ops']['x0_share_of_op_time']:.3f}", flush=True)

rec["sm_clock_after"] = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                                       text=True).stdout.strip()
rec["seconds"] = time.time() - t_start
rec["note"] = ("device_ms = CUDA events around one step on the current stream, the host waits for every step; ops = engine.prof "
               "(per-op CUDA events, eager coarse stack) in a separate run of its own; card = nvidia-smi name, power limit, max SM "
               "clock and SM clock at the start")
(out_dir / "h100_async_fusion.json").write_text(json.dumps(rec, indent=1))
print("wrote", out_dir / "h100_async_fusion.json")
