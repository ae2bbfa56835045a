"""Detection over a recorded sequence: SequenceDetector against the routes users have without it, in one process.

Config-5 shape: dagr-l at 640x480 on a 1 Mevents/s recording, 50 ms sliding windows every 1 ms over 2 s (the timed steps of
stream_benchmark), uniform and clustered.  Routes: StreamingDetector stepping through the recording (host wall clock and
device time per step, as stream_benchmark), and SequenceDetector.detect over the same windows at max_windows 8, 32, 64,
128 and 255 (host wall clock around detect(), which ends in a device synchronise; windows/s and gathered Mevents/s).
Hybrid: dagr-s + ResNet-50 at 640x480, a frame every 50 ms, interframe_windows(steps=10) over 2 s: one detect() against
per-window model(data) calls at B = 1.  Two rounds, routes alternated; the detections of the timed routes are asserted
equal on the timed data.  A separate torch.profiler run gives dagr_window_gather's device time and bytes / time.
Card name, power limit and clocks are read in the same run.  Writes OUT/h100_sequence.json
(usage: python tools/sequence_bench.py OUT)."""
import gc
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dagr_b200.data import EventBatch
from dagr_b200.model.dagr import DAGR
from dagr_b200.sequence import SequenceDetector, interframe_windows
from dagr_b200.streaming import StreamingDetector, _bench_setup, _latency, _timed_steps, synth_stream
from dagr_b200.utils.args import default_args
from tests.helpers import randomize_bn

W, H = 640, 480
RATE, CHUNK, WINDOW, SECONDS = 1_000_000, 1000, 50_000, 2.0
GS = (8, 32, 64, 128, 255)
GATHER_BYTES = 2 + 2 + 8 + 1 + 4 + 12 + 4          # read x, y, t, p; write batch, pos, feat (per gathered event)
HBM_TBS = 3.35                                       # H100 SXM data sheet

if len(sys.argv) != 2:
    sys.exit("usage: python tools/sequence_bench.py OUT_DIR")
out_dir = Path(sys.argv[1])
out_dir.mkdir(parents=True, exist_ok=True)
dev = torch.device("cuda:0")


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def same(a, b):
    return (len(a["boxes"]) == len(b["boxes"]) and torch.equal(a["boxes"].cpu(), b["boxes"].cpu())
            and torch.equal(a["scores"].cpu(), b["scores"].cpu()) and torch.equal(a["labels"].cpu(), b["labels"].cpu()))


def timed(fn):
    gc.collect()
    gc.disable()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    gc.enable()
    return r, ms


print("card (name, power limit, max SM clock, SM clock):", card(), flush=True)
torch.manual_seed(0)
dagr_l = randomize_bn(DAGR(default_args("l", batch_size=1), height=H, width=W).eval()).to(dev)

# ---- config-5 shape ----------------------------------------------------------------------------------------------------
streams = {}
for kind in ("uniform", "clustered"):
    _, evs, bounds, max_chunk = _bench_setup(dev, dagr_l, "l", W, H, 1, RATE, CHUNK, WINDOW, SECONDS, kind)
    warm = int(WINDOW / CHUNK) + 20                  # the steps _timed_steps does not time
    K = len(bounds[0]) - 1
    x, y, t, p = evs[0]
    t_end = (np.arange(warm, K) + 1) * CHUNK
    a, b = np.searchsorted(t, t_end - WINDOW), np.searchsorted(t, t_end)
    streams[kind] = dict(ev=dict(x=x, y=y, t=t, p=p), bounds=bounds, max_chunk=max_chunk, warm=warm, t_end=t_end,
                         gathered=int((b - a).sum()))


def stepping(kind):
    s = streams[kind]
    det = StreamingDetector(dagr_l, window_us=WINDOW, max_chunk=s["max_chunk"])
    res, orig = [], det.result
    det.result = lambda: res.append(orig()[0]) or res[-1]
    ev = s["ev"]
    lat, dev_ms, nev = _timed_steps(det, lambda c, te: det.submit(*c[0], te[0]), [(ev["x"], ev["y"], ev["t"], ev["p"])], s["bounds"],
                                    CHUNK, WINDOW)
    return _latency(lat, dev_ms, nev, CHUNK), res[s["warm"]:]


def sequence(kind, G):
    s = streams[kind]
    det = SequenceDetector(dagr_l, window_us=WINDOW, max_windows=G, max_events=(1 << 24) - 1)
    det.detect(s["ev"], s["t_end"][:2 * G])                                   # warm: geometry, workspace, captured coarse stack
    out, ms = timed(lambda: det.detect(s["ev"], s["t_end"]))
    Q = len(s["t_end"])
    return dict(max_windows=G, wall_ms=ms, ms_per_window=ms / Q, windows_per_s=Q / ms * 1e3,
                gathered_mev_s=s["gathered"] / ms / 1e3, windows=Q, gathered_events=s["gathered"]), out


records = []
for rnd in range(2):
    rec = dict(round=rnd, config5={})
    for kind in ("uniform", "clustered"):
        r = rec["config5"][kind] = dict(sequence=[])
        order = [None] + list(GS) if rnd == 0 else list(GS)[::-1] + [None]   # alternate the routes between rounds
        ref = None
        outs = {}
        for G in order:
            if G is None:
                r["stepping"], ref = stepping(kind)
                print(f"[{rnd}] {kind} stepping: host p50 {r['stepping']['latency_ms']['p50']:.3f} ms, device p50 "
                      f"{r['stepping']['device_ms']['p50']:.3f} ms per 1 ms step", flush=True)
            else:
                row, outs[G] = sequence(kind, G)
                r["sequence"].append(row)
                print(f"[{rnd}] {kind} detect G={G}: {row['wall_ms']:.1f} ms for {row['windows']} windows, {row['ms_per_window']:.3f} "
                      f"ms/window, {row['gathered_mev_s']:.0f} gathered Mev/s", flush=True)
        for G, out in outs.items():
            assert len(out) == len(ref) and all(same(a, b) for a, b in zip(out, ref)), (kind, G)
        r["sequence"].sort(key=lambda v: v["max_windows"])
        r["equal_to_stepping"] = True
    records.append(rec)

# ---- dagr_window_gather in a torch.profiler run of its own ---------------------------------------------------------------
prof_rows = {}
for kind in ("uniform", "clustered"):
    s = streams[kind]
    det = SequenceDetector(dagr_l, window_us=WINDOW, max_windows=64, max_events=(1 << 24) - 1)
    det.detect(s["ev"], s["t_end"][:128])
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        det.detect(s["ev"], s["t_end"])
        torch.cuda.synchronize()
    gather_us = device_us = 0.0
    n_gather = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        d = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "k_window_gather" in e.name:
            gather_us += d
            n_gather += 1
        if not e.name.startswith(("Memcpy", "Memset")) and "memcpy" not in e.name.lower():
            device_us += d
    nbytes = s["gathered"] * GATHER_BYTES
    prof_rows[kind] = dict(gather_launches=n_gather, gather_ms=gather_us / 1e3, kernels_ms=device_us / 1e3,
                           gather_share_of_kernel_time=gather_us / max(device_us, 1e-9), gathered_events=s["gathered"],
                           bytes=nbytes, tb_s=nbytes / (gather_us * 1e-6) / 1e12 if gather_us else None,
                           share_of_hbm_3_35_tb_s=(nbytes / (gather_us * 1e-6) / 1e12) / HBM_TBS if gather_us else None)
    print(f"profiler {kind}: gather {gather_us / 1e3:.2f} ms in {n_gather} launches = {prof_rows[kind]['gather_share_of_kernel_time'] * 100:.2f} % "
          f"of kernel time; {prof_rows[kind]['tb_s']:.2f} TB/s", flush=True)

# ---- hybrid: interframe windows -----------------------------------------------------------------------------------------
del streams
torch.manual_seed(0)
hybrid = randomize_bn(DAGR(default_args("s", batch_size=1, use_image=True, img_net="resnet50"), height=H, width=W).eval()).to(dev)
hx, hy, ht, hp = synth_stream(RATE, SECONDS + 0.06, W, H, seed=99, kind="uniform")
frame_t = np.arange(0, int(SECONDS * 1e6), 50_000)
g = torch.Generator().manual_seed(0)
frames = torch.randint(0, 256, (len(frame_t), 3, H, W), generator=g, dtype=torch.uint8)
tb, te, fi = interframe_windows(frame_t, steps=10, span_us=50_000)
hev = dict(x=hx, y=hy, t=ht, p=hp)


def per_window():
    out = []
    for q in range(len(te)):
        a, b = np.searchsorted(ht, [tb[q], te[q]])
        n = b - a
        pos = torch.from_numpy(np.stack([hx[a:b], hy[a:b], ht[a:b]], 1).astype(np.int32).reshape(n, 3)).to(dev)
        feat = torch.from_numpy(hp[a:b].astype(np.float32)).to(dev)
        d = EventBatch(x=feat.view(-1, 1), pos=torch.zeros(n, 3, device=dev), batch=torch.zeros(n, dtype=torch.long, device=dev),
                       width=torch.tensor([W]), height=torch.tensor([H]), time_window=torch.tensor([1_000_000]), pos_denorm=pos,
                       num_graphs=1, dims=(W, H, 1_000_000), image=frames[fi[q]].to(dev).float().unsqueeze(0) / 255.0)
        out.append(hybrid(d)[0][0])
    return out


hdet = SequenceDetector(hybrid, max_windows=64)
hdet.detect(hev, te[:128], t_begin=tb[:128], frames=frames, frame_idx=fi[:128])    # warm
per_window()
hyb = []
for rnd in range(2):
    row = dict(round=rnd)
    for route in (("sequence", "per_window") if rnd == 0 else ("per_window", "sequence")):
        if route == "sequence":
            out_s, row["sequence_ms"] = timed(lambda: hdet.detect(hev, te, t_begin=tb, frames=frames, frame_idx=fi))
        else:
            out_w, row["per_window_ms"] = timed(per_window)
    assert all(same(a, b) for a, b in zip(out_s, out_w))
    row.update(windows=len(te), frames=len(frame_t), speedup=row["per_window_ms"] / row["sequence_ms"], equal=True)
    print(f"[{rnd}] hybrid interframe: detect {row['sequence_ms']:.1f} ms, per-window model(data) {row['per_window_ms']:.1f} ms "
          f"({row['speedup']:.2f}x) for {len(te)} windows", flush=True)
    hyb.append(row)

res = dict(card_at_end=card(), config5_shape=dict(model="dagr-l", width=W, height=H, rate_mev_s=RATE / 1e6, window_us=WINDOW, step_us=CHUNK,
                                                  seconds=SECONDS, max_events=(1 << 24) - 1),
           rounds=records, window_gather_profile=prof_rows,
           hybrid=dict(model="dagr-s + resnet50", width=W, height=H, frame_us=50_000, interframe_steps=10, rounds=hyb),
           note="stepping = StreamingDetector, one chunk per 1 ms step submitted after the previous step's detections reached the host "
                "(stream_benchmark's loop): latency_ms = host wall clock per step, device_ms = CUDA events around the step.  sequence = "
                "one SequenceDetector.detect() over the same windows (t_end of every timed step, 50 ms sliding windows), host wall "
                "clock around the call including the upload of the host recording and both of its host syncs, after a warm-up call "
                "at the same max_windows; max_events = 2^24 - 1 so max_windows sets the block size.  gathered_mev_s = the events of "
                "all windows (each event counted once per window holding it) / wall time.  window_gather_profile = a separate "
                "torch.profiler run of one detect() at max_windows 64: the gather kernel's device time, its share of all kernel "
                "time, and 33 bytes per gathered event over its time.  hybrid = interframe_windows(steps=10) over 2 s with a frame "
                "every 50 ms: one detect() (each frame through the ResNet-50 trunk once) against one model(data) per window at B = "
                "1 from host arrays, the route without SequenceDetector.  The detections of every timed route are asserted equal.")
(out_dir / "h100_sequence.json").write_text(json.dumps(res, indent=1))
print("wrote", out_dir / "h100_sequence.json")
