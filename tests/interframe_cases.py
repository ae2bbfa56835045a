"""A synthetic DSEC-shaped recording with labels, for the interframe evaluation's tests and tools/interframe_eval_bench.py:
events, frames at a fixed rate and a DSEC tracks array (sensor pixel coordinates, labels at every frame) of boxes moving
with stable track ids, with births and deaths, occasional jumps (pairs the only-perfect-tracks rule drops), classes the
DSEC mapping drops, boxes leaving the frame, and frames without labels."""
import numpy as np

from dagr_b200.streaming import synth_stream

SOURCE = ("pedestrian", "rider", "car", "bus", "truck", "bicycle", "motorcycle", "train")
TRACK_DTYPE = np.dtype([("t", "<u8"), ("x", "<f4"), ("y", "<f4"), ("w", "<f4"), ("h", "<f4"), ("class_id", "u1"),
                        ("class_confidence", "<f4"), ("track_id", "<u4")])


def tracks_for(frame_t, seed, boxes=10, sensor=(640, 480)):
    """labels at every frame time (a few frames left without labels); box centres bounce off the sensor's edges"""
    rng = np.random.default_rng(seed)
    sw, sh = sensor
    rows, alive, next_id = [], {}, 1
    for f, t in enumerate(frame_t):
        for tid in [k for k in alive if rng.random() < 0.004]:                # deaths
            del alive[tid]
        while len(alive) < boxes:                                               # births
            w, h = rng.uniform(30, 200), rng.uniform(30, 160)
            alive[next_id] = dict(b=np.array([rng.uniform(-w / 2, sw - w / 2), rng.uniform(-h / 2, sh - h / 2), w, h]),
                                  v=rng.normal(0, 6, 2), c=int(rng.choice([0, 2, 2, 2, 3, 4, 1, 5])))
            next_id += 1
        if rng.random() < 0.01:
            continue                                                            # a frame without labels
        for tid, s in alive.items():
            s["b"][:2] += s["v"] + (rng.normal(0, 120, 2) if rng.random() < 0.003 else 0)
            c = s["b"][:2] + s["b"][2:] / 2
            s["v"] = np.where((c < 0) | (c > (sw, sh)), -s["v"], s["v"])      # bounce off the sensor's edges
            s["b"][2:] = np.maximum(s["b"][2:] * rng.uniform(0.97, 1.03, 2), 4)
            rows.append((int(t),) + tuple(float(v) for v in s["b"]) + (s["c"], 0.9, tid))
    tr = np.array(rows, dtype=TRACK_DTYPE)
    return tr[np.argsort(tr["t"], kind="stable")]


def recording(seconds, seed, width, height, rate=300_000, frame_us=50_000, sensor=None, t0=0, kind="clustered", boxes=10):
    """-> (events, frame_t int64, tracks).  Without sensor the events are at the model's width x height in the model's
    time base; with sensor=(sw, sh) they are raw camera events (t int64 from t0, p in {0, 1}).  Labels are in sensor
    pixels (2x the model's) either way."""
    sw, sh = sensor if sensor is not None else (2 * width, 2 * height)
    x, y, t, p = synth_stream(rate, seconds, sw if sensor is not None else width, sh if sensor is not None else height, seed=seed,
                              kind=kind)
    if sensor is None:
        events = dict(x=x, y=y, t=(t.astype(np.int64) + t0).astype(np.int32), p=p)
    else:
        events = dict(x=x.astype(np.uint16), y=y.astype(np.uint16), t=t.astype(np.int64) + t0, p=(p > 0).astype(np.int8))
    frame_t = t0 + np.arange(frame_us, int(seconds * 1e6) - frame_us, frame_us, dtype=np.int64)
    return events, frame_t, tracks_for(frame_t, seed, boxes, (sw, sh))
