"""The four stream benchmarks (stream_benchmark, the config-5 bench entry, multistream_benchmark, fusion_stream_benchmark and
fusion_multistream_benchmark), each run once at a small size: every result carries the same keys, and the fields that the
seeded streams fix -- timed steps, events per step, live events at the end, overflow, frames set during the timed steps --
equal what the chunk grid of the streams gives."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W, H, RATE, SECONDS, WINDOW, CHUNK, FRAME = 320, 215, 300_000, 0.1, 10_000, 1000, 20_000
KW = dict(size="n", width=W, height=H, rate_ev_s=RATE, chunk_us=CHUNK, window_us=WINDOW, seconds=SECONDS)

LATENCY = {"latency_ms", "device_ms", "sustained_mev_s", "realtime", "realtime_margin", "note"}
FUSION = {"latency_ms", "latency_ms_trunk_in_flight", "latency_ms_no_trunk", "device_ms", "trunk_device_ms", "frame_to_first_use_ms",
          "sustained_mev_s", "note"}
KEYS = dict(
    stream={"model", "stream_rate_mev_s", "chunk_us", "window_us", "stream_seconds", "chunks", "events_per_chunk", "live_events",
            "overflow"} | LATENCY,
    multistream={"model", "streams", "kind", "stream_rate_mev_s", "chunk_us", "window_us", "stream_seconds", "steps", "events_per_step",
                 "stage_bytes", "live_events", "overflow"} | LATENCY,
    fusion_stream={"model", "width", "height", "stream_rate_mev_s", "chunk_us", "window_us", "frame_us", "sync_frames", "step_priority",
                   "stream_seconds", "chunks", "frames", "events_per_chunk", "live_events", "overflow", "set_frame_host_ms"} | FUSION,
    fusion_multistream={"model", "streams", "width", "height", "stream_rate_mev_s", "chunk_us", "window_us", "frame_us", "frame_offset_us",
                        "stream_seconds", "steps", "frames", "events_per_step", "live_events", "overflow", "graphs",
                        "steps_trunk_in_flight"} | FUSION)


def _expected(S):
    """(timed steps, mean events per timed step, live events per stream after the last step, frames set in timed steps) of S
    streams (seeds 99, 100, ...) in CHUNK chunks, the first WINDOW / CHUNK + 20 steps untimed, camera s's frames every FRAME
    us from s * FRAME / S on."""
    from dagr_b200.streaming import synth_stream
    total_s = SECONDS + WINDOW * 1e-6 + 0.02
    grid = np.arange(0, int(total_s * 1e6) + CHUNK, CHUNK)
    warm = WINDOW // CHUNK + 20
    per_step, live = np.zeros(len(grid) - 1, np.int64), []
    for s in range(S):
        t = synth_stream(RATE, total_s, W, H, seed=99 + s)[2]
        b = np.searchsorted(t, grid)
        per_step += np.diff(b)
        live.append(int(b[-1] - np.searchsorted(t, grid[-1] - WINDOW)))          # t >= t_end - window of the last step
    offset = [(s * FRAME // S) // CHUNK * CHUNK for s in range(S)]
    frames = sum(1 for k in range(warm, len(grid) - 1) for o in offset if k * CHUNK > o and (k * CHUNK - o) % FRAME == 0)
    return len(grid) - 1 - warm, float(per_step[warm:].mean()), live, frames


@pytest.mark.parametrize("name", sorted(KEYS))
def test_stream_benchmark_fields(name):
    import torch
    from dagr_b200 import streaming
    dev = torch.device("cuda")
    S = 1 if name in ("stream", "fusion_stream") else 2
    fusion = dict(img_net="resnet18", frame_us=FRAME) if name.startswith("fusion") else {}
    bench = getattr(streaming, f"{name}_benchmark")
    r = bench(dev, S, **KW, **fusion) if S > 1 else bench(dev, **KW, **fusion)
    assert set(r) == KEYS[name]
    steps, per_step, live, frames = _expected(S)
    key = "chunk" if S == 1 else "step"
    assert r[f"{key}s"] == steps and r[f"events_per_{key}"] == pytest.approx(per_step, rel=1e-12)
    assert r["live_events"] == (live[0] if S == 1 else live)
    assert r["overflow"] == (False if S == 1 else [False] * S)
    if fusion:
        assert r["frames"] == frames > 0
        assert set(r["latency_ms"]) == {"n", "p50", "p99", "max"} and r["latency_ms"]["n"] == steps
    else:
        assert set(r["latency_ms"]) == {"p50", "p90", "p99", "max"} and set(r["device_ms"]) == {"p50", "p99"}
    if name == "fusion_multistream":
        assert r["graphs"] == 1 and len(r["frame_to_first_use_ms"]) == S
