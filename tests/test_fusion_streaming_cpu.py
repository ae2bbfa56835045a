"""Fusion streaming front end without a GPU: the constructor checks of FusionStreamingDetector (they run before any device
work) and the argument contract of dagr_l1_x0_image_live (every null pointer is refused with DAGR_E_ARG and a message before
anything is launched)."""
import ctypes as C

import pytest

from tests.helpers import make_model

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first


def test_fusion_detector_refuses_events_only_and_no_events_models():
    from dagr_b200.streaming import FusionStreamingDetector
    events_only, _ = make_model("n", 180, 240)
    with pytest.raises(ValueError, match="StreamingDetector"):
        FusionStreamingDetector(events_only)
    image_only, _ = make_model("n", 180, 240, use_image=True, img_net="resnet18", no_events=True)
    with pytest.raises(NotImplementedError, match="no event path"):
        FusionStreamingDetector(image_only)


@pytest.mark.parametrize("null", ["g", "start", "xyb", "img0", "x0"])
def test_x0_image_live_rejects_null_pointers(null):
    from dagr_b200 import _lib
    from dagr_b200.geometry import Geometry
    lib = _lib.load()
    geom = Geometry(240, 180, 1, device="cpu")
    a = dict(g=C.byref(geom.c_geom), start=BAD, xyb=BAD, img0=BAD, x0=BAD)
    a[null] = None
    rc = lib.dagr_l1_x0_image_live(a["g"], 1 << 10, a["start"], a["xyb"], None, a["img0"], 8, 8, a["x0"], None)
    assert rc == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_l1_x0_image_live" in msg and "null" in msg, msg


def test_x0_image_live_rejects_out_of_range_n():
    from dagr_b200 import _lib
    from dagr_b200.geometry import Geometry
    lib = _lib.load()
    geom = Geometry(240, 180, 1, device="cpu")
    assert lib.dagr_l1_x0_image_live(C.byref(geom.c_geom), -1, BAD, BAD, None, BAD, 8, 8, BAD, None) == E_ARG
    assert "N out of range" in lib.dagr_last_error().decode()
