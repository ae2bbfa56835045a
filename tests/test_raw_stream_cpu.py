"""Raw sensor streaming without a GPU: the host packing of the raw stage, the argument contract of dagr_stream_ingest (every
bad input is refused with DAGR_E_ARG and a message before anything is launched) and the detectors' construction checks."""
import ctypes as C

import numpy as np
import pytest

from tests.helpers import make_model

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first


def _chunk(rng, n, t0, p01=True):
    return (rng.integers(0, 640, n).astype(np.uint16), rng.integers(0, 480, n).astype(np.uint16),
            (t0 + np.sort(rng.integers(0, 1000, n))).astype(np.int64),
            rng.integers(0, 2, n).astype(np.int8) if p01 else rng.choice([-1, 1], n).astype(np.int8))


def test_pack_raw_stage_round_trips():
    from dagr_b200.streaming import pack_raw_stage
    S, mr = 4, 7
    rng = np.random.default_rng(0)
    chunks = [_chunk(rng, 3, -5), None, _chunk(rng, 7, 2_000_000_000, p01=False), _chunk(rng, 0, 0)]
    chunks[0][0][0], chunks[0][1][0] = 65535, 32767                  # the widest coordinates the record holds
    stage = np.full(4 * S + 2 * S * mr, -7, dtype=np.int32)
    ns = pack_raw_stage(stage, chunks, [10, -20, 30, -(1 << 31)], mr, planes=[0, 3, 5, 1])
    assert ns == [3, 0, 7, 0]
    assert stage[:4 * S].reshape(S, 4).tolist() == [[3, 10, 0, 0], [0, -20, 3, 3], [7, 30, 3, 5], [0, -(1 << 31), 10, 1]]
    ev = stage[4 * S:].reshape(-1, 2)
    for s, o in ((0, 0), (2, 3)):
        x, y, t, p = chunks[s]
        w = ev[o:o + len(t), 0].view(np.uint32)
        assert np.array_equal(w & 0xffff, x) and np.array_equal((w >> 16) & 0x7fff, y)
        assert np.array_equal((w >> 31).astype(np.int8), (p > 0).astype(np.int8))
        assert np.array_equal(2 * (w >> 31).astype(np.int32) - 1, np.where(p > 0, 1, -1))   # the 2p - 1 the kernel applies
        assert np.array_equal(ev[o:o + len(t), 1], t.astype(np.int32))
    assert (ev[10:] == -7).all()                       # nothing written behind the last stream's events
    plain = np.zeros_like(stage)
    pack_raw_stage(plain, chunks, [10, -20, 30, 0], mr)
    assert plain[3:4 * S:4].tolist() == [0, 0, 0, 0]     # no planes: word 3 is 0
    with pytest.raises(ValueError, match="max_raw"):
        pack_raw_stage(stage, [_chunk(rng, 8, 0), None, None, None], [0] * 4, mr)
    with pytest.raises(ValueError, match="smaller"):
        pack_raw_stage(stage[:-1], chunks, [0] * 4, mr)


def _ingest(lib, raw=BAD, streams=2, max_raw=4096, fx=2, fy=2, ow=320, oh=240, crop=215, cmap=BAD, stage=BAD, max_chunk=4096):
    return lib.dagr_stream_ingest(raw, streams, max_raw, fx, fy, ow, oh, crop, cmap, stage, max_chunk, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(raw=None), "null"),
    (dict(cmap=None), "null"),
    (dict(stage=None), "null"),
    (dict(streams=0), "streams"),
    (dict(streams=128), "streams"),
    (dict(fx=0), "fx"),
    (dict(fy=0), "fx"),
    (dict(ow=32769, fx=2), "geometry"),
    (dict(oh=16385, fy=2), "geometry"),
    (dict(ow=640, oh=480), "2^18"),
    (dict(crop=0), "crop_h"),
    (dict(crop=241), "crop_h"),
    (dict(max_raw=0), "max_raw"),
    (dict(max_raw=16385, max_chunk=1 << 15), "max_raw"),
    (dict(max_raw=4096, max_chunk=4095), "max_chunk"),
])
def test_stream_ingest_rejects_bad_arguments(kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _ingest(lib, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_stream_ingest" in msg and needle in msg, msg


def test_stream_ingest_limits_match_the_host_constants():
    from dagr_b200 import streaming
    from pathlib import Path
    h = (Path(__file__).resolve().parent.parent / "include" / "dagr_b200.h").read_text()
    assert "#define DAGR_INGEST_MAX_RAW   16384" in h and streaming.MAX_RAW == 16384
    assert "#define DAGR_INGEST_MAX_CELLS (1 << 18)" in h and streaming.MAX_CELLS == 1 << 18


def test_raw_detectors_check_the_sensor_before_anything_else():
    from dagr_b200.streaming import MultiStreamDetector, StreamingDetector
    model, _ = make_model("n", 215, 320)
    for kw, needle in [(dict(sensor=(641, 480)), "integer multiple"), (dict(sensor=(640, 429)), "integer multiple"),
                       (dict(sensor=(160, 480)), "integer multiple"), (dict(sensor=(640, 480), max_chunk=16385), "max_chunk"),
                       (dict(sensor=(640, 2048)), "2\\^18"), (dict(sensor=(640 * 256, 480 * 256)), "2\\^16"),
                       (dict(p_is_01=False), "sensor")]:
        with pytest.raises(ValueError, match=needle):
            StreamingDetector(model, **kw)
        with pytest.raises(ValueError, match=needle):
            MultiStreamDetector(model, streams=2, **kw)
    # a valid sensor gets as far as the device check (the model is on the CPU)
    with pytest.raises(RuntimeError, match="CUDA"):
        StreamingDetector(model, sensor=(640, 480))
