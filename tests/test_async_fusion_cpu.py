"""Incremental updates of the image-fusion model without a GPU: the refusals of AsyncDAGR that happen before any device
work (--no_events, a first step without a frame), and the argument contract of the two incremental entry points
dagr_l1_conv_a_image_inc / dagr_voxel_sample_max_inc (every bad argument is refused with DAGR_E_ARG and a message before
anything is launched)."""
import ctypes as C

import pytest
import torch

from tests.helpers import make_inputs, make_model

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first
W, H = 240, 180


def test_async_refuses_no_events_model():
    from dagr_b200.asynchronous import AsyncDAGR
    image_only, _ = make_model("n", H, W, use_image=True, img_net="resnet18", no_events=True)
    with pytest.raises(NotImplementedError, match="no event path"):
        AsyncDAGR(image_only)


def test_async_first_step_without_a_frame_is_refused():
    from dagr_b200.asynchronous import AsyncDAGR
    model, _ = make_model("n", H, W, use_image=True, img_net="resnet18")
    _, data = make_inputs(1, 500, W, H, seed=3)
    assert getattr(data, "image", None) is None
    a = AsyncDAGR(model)
    with pytest.raises(ValueError, match="needs chunk.image"):
        a.step_decoded(data, batch_size=1)                       # the events stay on the CPU: nothing reached a device
    data.image = torch.zeros(2, 3, H, W)
    with pytest.raises(ValueError, match="expected a formatted float"):
        a.step_decoded(data, batch_size=1)                       # a frame of the wrong batch size


_PARAMS = []                   # keeps the host-side parameter structs alive while their byref() is in use


def _conv_a_args(geom):
    from dagr_b200 import _lib
    _PARAMS.append(_lib.L1ImgParams())
    return dict(g=C.byref(geom.c_geom), start=BAD, xyb=BAD, ti=BAD, feat_s=BAD, x0=BAD, nbr=BAD, off=BAD, p_host=C.byref(_PARAMS[-1]),
                wfrag=BAD, xa=BAD, skipv=BAD)


def _conv_a(lib, a, N=1 << 10, min_idx=1):
    return lib.dagr_l1_conv_a_image_inc(a["g"], N, a["start"], a["xyb"], a["ti"], a["feat_s"], a["x0"], a["nbr"], a["off"],
                                        a["p_host"], a["wfrag"], min_idx, a["xa"], a["skipv"], None, None, 0, None)


def _sample_args(geom):
    return dict(g=C.byref(geom.c_geom), start=BAD, xyb=BAD, ti=BAD, img=BAD, persist=BAD, xg=BAD)


def _sample(lib, a, N=1 << 10, min_idx=1, C_=64, ldx=80, c0=16, pool_mean=0):
    return lib.dagr_voxel_sample_max_inc(a["g"], N, a["start"], a["xyb"], a["ti"], a["img"], C_, 8, 8, min_idx, a["persist"], a["xg"],
                                         ldx, c0, pool_mean, None)


def _lib_geom():
    from dagr_b200 import _lib
    from dagr_b200.geometry import Geometry
    return _lib.load(), Geometry(W, H, 1, device="cpu")


@pytest.mark.parametrize("null", ["g", "start", "xyb", "ti", "feat_s", "x0", "nbr", "off", "p_host", "wfrag", "xa", "skipv"])
def test_conv_a_image_inc_rejects_null_pointers(null):
    lib, geom = _lib_geom()
    a = _conv_a_args(geom)
    a[null] = None
    assert _conv_a(lib, a) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_l1_conv_a_image_inc" in msg and "null" in msg, msg


def test_conv_a_image_inc_rejects_bad_min_idx_and_n():
    lib, geom = _lib_geom()
    assert _conv_a(lib, _conv_a_args(geom), min_idx=-1) == E_ARG
    assert "min_idx" in lib.dagr_last_error().decode()
    for n in (-1, 1 << 31):
        assert _conv_a(lib, _conv_a_args(geom), N=n) == E_ARG
        assert "N out of range" in lib.dagr_last_error().decode()


@pytest.mark.parametrize("null", ["g", "start", "xyb", "ti", "img", "persist", "xg"])
def test_voxel_sample_max_inc_rejects_null_pointers(null):
    lib, geom = _lib_geom()
    a = _sample_args(geom)
    a[null] = None
    assert _sample(lib, a) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_voxel_sample_max_inc" in msg and "null" in msg, msg


def test_voxel_sample_max_inc_rejects_bad_arguments():
    lib, geom = _lib_geom()
    for kw, what in ((dict(min_idx=-1), "min_idx"), (dict(N=-1), "N out of range"), (dict(N=1 << 31), "N out of range"),
                     (dict(c0=17), "ldx"), (dict(C_=65), "ldx"), (dict(pool_mean=1), "pool_mean")):
        assert _sample(lib, _sample_args(geom), **kw) == E_ARG, kw
        msg = lib.dagr_last_error().decode()
        assert "dagr_voxel_sample_max_inc" in msg and what in msg, (kw, msg)
