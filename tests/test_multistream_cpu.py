"""Multi-stream streaming front end without a GPU: the argument contract of dagr_stream_push_multi / dagr_graph_sort_rings
(every bad input is refused with DAGR_E_ARG and a message before anything is launched), the host-side packing of the
multi-stream stage, and the construction-time checks of MultiStreamDetector."""
import ctypes as C

import numpy as np
import pytest

from tests.helpers import make_model

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first


def _push(lib, ctl=BAD, stage=BAD, capacity=1 << 10, streams=2, max_chunk=256):
    return lib.dagr_stream_push_multi(ctl, stage, BAD, BAD, BAD, capacity, streams, max_chunk, None)


def _sort(lib, geom, capacity=1 << 10, streams=2, ctl=BAD):
    return lib.dagr_graph_sort_rings(C.byref(geom.c_geom), BAD, BAD, BAD, capacity, streams, ctl, BAD, BAD, BAD, BAD, BAD, BAD, BAD,
                                     BAD, BAD, None, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(capacity=1000), "power of two"),
    (dict(capacity=1 << 10, max_chunk=2048), "max_chunk"),
    (dict(streams=0), "streams"),
    (dict(streams=128), "streams"),
    (dict(streams=2, capacity=1 << 23), "2^24"),
    (dict(streams=64, capacity=1 << 18), "2^24"),
    (dict(ctl=None), "null"),
    (dict(stage=None), "null"),
])
def test_stream_push_multi_rejects_bad_arguments(kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _push(lib, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_stream_push_multi" in msg and needle in msg, msg


@pytest.mark.parametrize("kw,B,needle", [
    (dict(capacity=1000), 2, "power of two"),
    (dict(streams=0), 2, "streams"),
    (dict(streams=3), 2, "batch size"),
    (dict(streams=2, capacity=1 << 23), 2, "2^24"),
    (dict(ctl=None), 2, "null"),
])
def test_graph_sort_rings_rejects_bad_arguments(kw, B, needle):
    from dagr_b200 import _lib
    from dagr_b200.geometry import Geometry
    lib = _lib.load()
    geom = Geometry(240, 180, B, device="cpu")
    assert _sort(lib, geom, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_graph_sort_rings" in msg and needle in msg, msg


def test_pack_stage_header_offsets_and_empty_chunks():
    from dagr_b200.streaming import pack_stage
    S, mc = 4, 5
    rng = np.random.default_rng(0)

    def chunk(n, t0):
        return (rng.integers(0, 240, n).astype(np.int16), rng.integers(0, 180, n).astype(np.int16),
                (t0 + np.arange(n)).astype(np.int32), rng.choice([-1, 1], n).astype(np.int8))

    chunks = [chunk(3, 100), None, chunk(5, 7_000_000), chunk(0, 0)]
    stage = np.full(4 * S + 4 * S * mc, -7, dtype=np.int32)
    ns = pack_stage(stage, chunks, [10, 20, 30, 40], mc)
    assert ns == [3, 0, 5, 0]
    assert stage[:4 * S].reshape(S, 4).tolist() == [[3, 10, 0, 0], [0, 20, 3, 0], [5, 30, 3, 0], [0, 40, 8, 0]]
    ev = stage[4 * S:].reshape(-1, 4)
    for s, o in ((0, 0), (2, 3)):
        x, y, t, p = chunks[s]
        assert np.array_equal(ev[o:o + len(t)], np.stack([x, y, t, p], 1).astype(np.int32))
    assert (ev[8:] == -7).all()                        # nothing written behind the last stream's events
    with pytest.raises(ValueError, match="max_chunk"):
        pack_stage(stage, [chunk(6, 0), None, None, None], [0] * 4, mc)


def test_multistream_detector_rejects_image_fusion_and_oversized_rings():
    from dagr_b200.streaming import MultiStreamDetector
    img, _ = make_model("n", 180, 240, use_image=True, img_net="resnet18")
    with pytest.raises(NotImplementedError, match="events-only"):
        MultiStreamDetector(img, streams=2)
    model, _ = make_model("n", 180, 240)
    with pytest.raises(ValueError, match="2\\^24"):
        MultiStreamDetector(model, streams=128 // 2, capacity=1 << 18)
    with pytest.raises(ValueError, match="2\\^24"):
        MultiStreamDetector(model, streams=127, capacity=1 << 17 | 1)      # rounds up to 2^18 per stream
    with pytest.raises(ValueError, match="streams"):
        MultiStreamDetector(model, streams=0)
    with pytest.raises(ValueError, match="max_chunk"):
        MultiStreamDetector(model, streams=2, capacity=1 << 10, max_chunk=4096)
