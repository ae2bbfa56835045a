"""CPU restatement of the reference's event ingest (TEST INFRASTRUCTURE ONLY -- never imported by the product path).

Follows, line by line:
  * scripts/downsample_events.py:91-124  downsample_events / _filter_events_resize (2x event down-sampler: a signed
    accumulator per output pixel, an event passes when the accumulator reaches +-1 and is then reset by -p)
  * src/dagr/data/dsec_data.py:141-147,177-179  window slice `t < t_cut`, crop `y < height`, t relative to the last
    kept event, polarity 2p-1
  * src/dagr/data/utils.py:6-20 (int16 / int32 casts), src/dagr/utils/buffers.py:33-44 (true division by [W,H,T] in
    fp32), src/dagr/model/layers/ev_tgn.py:11-16 ((pos*[W,H,T]+1e-3).int())

Pinned by tests/golden/downsample_golden.npz, generated in the build container from the reference's own numba
function (tests/golden/make_downsample_golden.py), and by tests/golden/ingest_window_golden.npz, generated from the
reference's own preprocess_events / to_data / format_data / denormalize_pos (tests/golden/make_ingest_window_golden.py);
tests/test_ingest_kernels_cpu.py checks preprocess_window against it bit for bit.
"""
import numpy as np


def filter_events_resize(x, y, p, change_map, fx, fy):
    """scripts/downsample_events.py:109-124.  change_map float32[out_h,out_w] is updated in place; returns bool mask.
    numba semantics of `a[idx] += p*1.0/(fx*fy)` on a float32 array: the sum is formed in float64, stored as float32;
    `a[idx] -= p` with int8 p is float32 arithmetic."""
    mask = np.zeros(len(x), dtype=bool)
    d = float(fx * fy)
    for i in range(len(x)):
        xl, yl = int(x[i]) // fx, int(y[i]) // fy
        v = np.float32(np.float64(change_map[yl, xl]) + np.float64(p[i]) * 1.0 / d)
        if abs(v) >= 1:
            mask[i] = True
            v = np.float32(v - np.float32(p[i]))
        change_map[yl, xl] = v
    return mask


def downsample_events(events, input_height, input_width, output_height, output_width, change_map=None):
    """scripts/downsample_events.py:91-106.  events: dict of x (u16), y (u16), p (int8, +-1), t; returns (events, map)."""
    if change_map is None:
        change_map = np.zeros((output_height, output_width), dtype="float32")
    fx, fy = int(input_width / output_width), int(input_height / output_height)
    mask = filter_events_resize(events["x"], events["y"], events["p"], change_map, fx, fy)
    out = {k: v[mask] for k, v in events.items()}
    out["x"] = (out["x"] / fx).astype("uint16")
    out["y"] = (out["y"] / fy).astype("uint16")
    return out, change_map


def preprocess_window(events, width, height, time_window, t_cut=None):
    """dsec_data.py:177-179 then :141-147 then data/utils.py:6-20, buffers.py:33-44 and ev_tgn.py:11-16:
    raw (x, y, t us, p in {0,1}) -> pos_denorm int32[M,3], polarity float32[M].  t[-1] is the t of the last kept event in
    array order, whatever the order or sign of the timestamps."""
    ev = dict(events)
    if t_cut is not None:
        keep = ev["t"] < t_cut
        ev = {k: v[keep] for k, v in ev.items()}
    keep = ev["y"] < height
    ev = {k: v[keep] for k, v in ev.items()}
    t = ev["t"].astype(np.int64)
    if len(t) > 0:
        t = time_window + t - t[-1]
    pol = (2 * ev["p"].astype("int8") - 1).astype(np.float32)
    xy = np.stack([ev["x"], ev["y"]], axis=-1).astype("int16")
    pos = np.concatenate([xy.astype(np.int32), t.astype("int32").reshape(-1, 1)], axis=1)
    norm = np.array([width, height, time_window], dtype=np.float32)
    posf = pos.astype(np.float32) / norm                               # torch int / int -> fp32 true division
    den = (posf * norm + np.float32(1e-3)).astype(np.int32)             # separate fp32 multiply and add, truncation
    return den, pol
