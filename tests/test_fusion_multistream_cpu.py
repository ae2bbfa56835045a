"""Multi-camera fusion streaming front end without a GPU: the constructor checks of FusionMultiStreamDetector (they run
before any device work), the argument contract of the four *_planes entry points (every bad input is refused with
DAGR_E_ARG and a message naming the entry point before anything is launched), and the plane word of the packed stage."""
import ctypes as C

import numpy as np
import pytest

from tests.helpers import make_model

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first


def test_fusion_multistream_detector_refuses_events_only_no_events_and_bad_limits():
    from dagr_b200.streaming import FusionMultiStreamDetector, FusionStreamingDetector
    events_only, _ = make_model("n", 180, 240)
    with pytest.raises(ValueError, match="MultiStreamDetector"):
        FusionMultiStreamDetector(events_only, streams=2)
    image_only, _ = make_model("n", 180, 240, use_image=True, img_net="resnet18", no_events=True)
    with pytest.raises(NotImplementedError, match="no event path"):
        FusionMultiStreamDetector(image_only, streams=2)
    model, _ = make_model("n", 180, 240, use_image=True, img_net="resnet18")
    with pytest.raises(ValueError, match="streams"):
        FusionMultiStreamDetector(model, streams=0)
    with pytest.raises(ValueError, match="streams"):
        FusionMultiStreamDetector(model, streams=128)
    with pytest.raises(ValueError, match="2\\^24"):
        FusionMultiStreamDetector(model, streams=64, capacity=1 << 18)
    with pytest.raises(ValueError, match="max_chunk"):
        FusionMultiStreamDetector(model, streams=2, capacity=1 << 10, max_chunk=4096)
    # the one-camera detector takes the same construction checks
    with pytest.raises(ValueError, match="2\\^24"):
        FusionStreamingDetector(model, capacity=1 << 24)
    with pytest.raises(ValueError, match="2\\^24"):
        FusionStreamingDetector(model, capacity=(1 << 23) + 1)            # rounds up to 2^24
    with pytest.raises(ValueError, match="max_chunk"):
        FusionStreamingDetector(model, capacity=1 << 10, max_chunk=4096)


def test_multistream_detector_still_refuses_fusion_models():
    from dagr_b200.streaming import MultiStreamDetector
    model, _ = make_model("n", 180, 240, use_image=True, img_net="resnet18")
    with pytest.raises(NotImplementedError, match="events-only"):
        MultiStreamDetector(model, streams=2)


def _geom(B=2):
    from dagr_b200.geometry import Geometry
    return Geometry(240, 180, B, device="cpu")


def _x0(lib, a, N=1 << 10, nplanes=4, stride=4, h=8, w=8, C=64, ld=80):
    return lib.dagr_l1_x0_image_planes(a["g"], N, a["start"], a["xyb"], None, a["img"], h, w, nplanes, a["plane"], stride, a["out"],
                                       None)


def _vox(lib, a, N=1 << 10, nplanes=4, stride=4, h=8, w=8, C=64, ld=80):
    return lib.dagr_voxel_sample_max_planes(a["g"], N, a["start"], a["xyb"], a["img"], C, h, w, nplanes, a["plane"], stride, a["out"],
                                            ld, 16, 0, None)


def _sample(lib, a, N=1 << 10, nplanes=4, stride=4, h=8, w=8, C=64, ld=80):
    return lib.dagr_sample_features_planes(a["img"], nplanes, a["plane"], stride, C, h, w, a["posx"], a["posy"], a["bidx"], N, 240,
                                           180, a["out"], ld, 16, None)


def _head(lib, a, N=None, nplanes=4, stride=4):
    return lib.dagr_head_finish_planes(a["gr"], a["cnt"], a["cls"], 2, a["regobj"], 5, a["add_cls"], a["add_reg"], a["add_obj"], 2,
                                       32, 0, 100, nplanes, a["plane"], stride, a["out"], None)


ENTRY = dict(dagr_l1_x0_image_planes=(_x0, ["g", "start", "xyb", "img", "plane", "out"]),
             dagr_voxel_sample_max_planes=(_vox, ["g", "start", "xyb", "img", "plane", "out"]),
             dagr_sample_features_planes=(_sample, ["img", "plane", "posx", "posy", "bidx", "out"]),
             dagr_head_finish_planes=(_head, ["gr", "cnt", "cls", "regobj", "add_cls", "add_reg", "add_obj", "plane", "out"]))


def _args(geom):
    a = {k: BAD for k in ("start", "xyb", "img", "plane", "out", "posx", "posy", "bidx", "cnt", "cls", "regobj", "add_cls", "add_reg",
                          "add_obj")}
    a["g"] = C.byref(geom.c_geom)
    a["gr"] = C.byref(geom.levels[3].grid)
    return a


@pytest.mark.parametrize("name,null", [(n, p) for n, (_, ps) in ENTRY.items() for p in ps])
def test_planes_entry_points_reject_null_pointers(name, null):
    from dagr_b200 import _lib
    lib = _lib.load()
    geom = _geom()
    call, _ = ENTRY[name]
    a = _args(geom)
    a[null] = None
    assert call(lib, a) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert name in msg and "null" in msg, msg


COUNTS = [(dict(nplanes=0), "nplanes"), (dict(nplanes=-3), "nplanes"), (dict(stride=0), "plane_stride"), (dict(stride=-4), "plane_stride")]
EVENTS = [(dict(N=-1), "N out of range"), (dict(N=1 << 31), "N out of range")]          # dagr_head_finish_planes takes no count
# the sampling forms' maps and rows (c0 = 16): h, w >= 1 and the channels [c0, c0 + C) within the row stride
MAPS = [(dict(h=0), "h, w >= 1"), (dict(w=0), "h, w >= 1")]
ROWS = {"dagr_voxel_sample_max_planes": [(dict(ld=79), "ldx")], "dagr_sample_features_planes": [(dict(ld=79), "ldo"), (dict(C=0), "C, h, w")]}


@pytest.mark.parametrize("name,kw,needle", [(n, kw, m) for n in sorted(ENTRY) for kw, m in COUNTS + (EVENTS if "head" not in n else [])]
                         + [(n, kw, m) for n in sorted(ENTRY) for kw, m in (MAPS if "head" not in n else []) + ROWS.get(n, [])])
def test_planes_entry_points_reject_bad_counts(name, kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    geom = _geom()
    call, _ = ENTRY[name]
    assert call(lib, _args(geom), **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert name in msg and needle in msg, msg


def test_voxel_sample_max_planes_rejects_channels_past_the_row():
    from dagr_b200 import _lib
    lib = _lib.load()
    geom = _geom()
    a = _args(geom)
    assert lib.dagr_voxel_sample_max_planes(a["g"], 1 << 10, BAD, BAD, BAD, 64, 8, 8, 4, BAD, 4, BAD, 79, 16, 0, None) == E_ARG
    assert "ldx" in lib.dagr_last_error().decode()


def test_pack_stage_writes_planes_into_word_3():
    from dagr_b200.streaming import pack_stage
    S, mc = 3, 4
    chunks = [(np.array([1, 2], np.int16), np.array([3, 4], np.int16), np.array([10, 11], np.int32), np.array([1, -1], np.int8)),
              None, (np.array([5], np.int16), np.array([6], np.int16), np.array([7], np.int32), np.array([1], np.int8))]
    plain = np.full(4 * S + 4 * S * mc, -7, dtype=np.int32)
    pack_stage(plain, chunks, [100, 200, 300], mc)
    assert plain[:4 * S].reshape(S, 4).tolist() == [[2, 100, 0, 0], [0, 200, 2, 0], [1, 300, 2, 0]]
    planes = np.full_like(plain, -7)
    pack_stage(planes, chunks, [100, 200, 300], mc, planes=[1, 2, 5])
    assert planes[:4 * S].reshape(S, 4).tolist() == [[2, 100, 0, 1], [0, 200, 2, 2], [1, 300, 2, 5]]
    assert np.array_equal(planes[4 * S:], plain[4 * S:])           # the events are packed as without planes
