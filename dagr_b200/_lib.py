"""ctypes binding of libdagr_b200.so (the C-ABI declared in include/dagr_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, a
RuntimeError is raised (the reference raises RuntimeError from AT_ASSERTM the same way,
src/dagr/graph/ev_graph.cu:9-12).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parent
# DAGR_B200_LIB points at an alternative build of the same sources (kernel A/B experiments, tools/ab_build.py)
_LIB_PATH = Path(os.environ["DAGR_B200_LIB"]) if os.environ.get("DAGR_B200_LIB") else _PKG / "libdagr_b200.so"
_lib = None

ELL = 16
KU = 15
TABW = 16
L1_TC_WFRAG_FLOATS = 8192               # DAGR_L1_TC_WFRAG_FLOATS
L1A_TC_WFRAG_FLOATS = 1536              # DAGR_L1A_TC_WFRAG_FLOATS

p = C.c_void_p
i32 = C.c_int32
i64 = C.c_int64
f32 = C.c_float
_Tensor = torch.Tensor
_void_p = C.c_void_p.from_param


class Dev:
    """argument type of a device pointer (the header's convention: every pointer not named *_host).  A CUDA tensor passes
    its data_ptr() and stays alive through the call; None passes NULL; raw addresses (int, c_void_p) pass unchanged.  A
    tensor in host memory, pinned or not, is refused before the call: a kernel would fault on it or read it over PCIe."""

    @staticmethod
    def from_param(obj):
        if isinstance(obj, _Tensor):
            if not obj.is_cuda:
                raise RuntimeError(f"a {obj.device} tensor where the library takes a device pointer")
            return _void_p(obj.data_ptr())
        return _void_p(obj)


class Host:
    """argument type of a *_host pointer: host memory (ctypes arrays and buffers), never a CUDA tensor."""

    @staticmethod
    def from_param(obj):
        if getattr(obj, "is_cuda", False):
            raise RuntimeError("a CUDA tensor where the library takes a host pointer")
        return _void_p(obj)


class Geom(C.Structure):
    _fields_ = [("W", i32), ("H", i32), ("B", i32), ("T", i32),
                ("r", i32), ("ncell", i32),
                ("dt_us", i32), ("K", i32), ("Q", i32),
                ("nx1", i32), ("ny1", i32),
                ("CW", i32), ("CH", i32), ("CP", i32),
                ("NK", i32),
                ("xkey", p), ("ykey", p), ("spiral", p), ("posx0", p), ("posy0", p), ("vx0", p), ("vy0", p), ("tabx", p), ("taby", p)]


class Grid(C.Structure):
    _fields_ = [("nx", i32), ("ny", i32), ("B", i32), ("W", i32), ("H", i32),
                ("posxr", p), ("posyr", p)]


class EventWs(C.Structure):
    _fields_ = [(k, i64) for k in ("key", "tmp", "count", "blocksums", "start", "perm", "ti", "xyb", "feat_s", "nbr", "off", "cellmask",
                                   "xa", "wl_hdr", "wl_ids", "x1")]


class PoolWs(C.Structure):
    _fields_ = [(k, i64) for k in ("acc", "possum", "ptmax", "pcnt", "pmask")]


class EvalParams(C.Structure):
    _fields_ = [("iou_thrs", C.c_double * 10), ("rec_thrs", C.c_double * 101), ("area_rng", C.c_double * 8)]


class L1AParams(C.Structure):
    _fields_ = [("w", f32 * (KU * 3 * 16)), ("root", f32 * (3 * 16)),
                ("scale", f32 * 16), ("shift", f32 * 16), ("relu", i32)]


class L1ImgParams(C.Structure):
    _fields_ = [("w", f32 * (KU * 24 * 16)), ("root", f32 * (24 * 16)), ("skip", f32 * (24 * 16)),
                ("scale", f32 * 16), ("shift", f32 * 16), ("sscale", f32 * 16), ("sshift", f32 * 16), ("relu", i32)]


class L1BParams(C.Structure):
    _fields_ = [("w", f32 * (KU * 16 * 16)), ("root", f32 * (16 * 16)), ("skip", f32 * (3 * 16)),
                ("scale", f32 * 16), ("shift", f32 * 16), ("sscale", f32 * 16), ("sshift", f32 * 16),
                ("relu", i32), ("pool_mean", i32), ("xs", i32 * 3), ("ys", i32 * 5), ("den_x", f32), ("den_y", f32)]


_SIGS = {
    "dagr_abi_version": (C.c_int, []),
    "dagr_last_error": (C.c_char_p, []),
    "dagr_scan_blocks": (i64, [i64]),
    "dagr_check_config": (C.c_int, [C.POINTER(Geom), i64, C.c_int, C.c_int, C.c_char_p]),
    "dagr_event_workspace_bytes": (C.c_int, [C.POINTER(Geom), i64, C.POINTER(EventWs)]),
    "dagr_pool_workspace_bytes": (C.c_int, [i64, C.c_int, C.POINTER(PoolWs)]),
    "dagr_downsample_events": (C.c_int, [Dev, Dev, Dev, i64, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev, Dev, Dev, Dev, Dev,
                                         Dev, Dev, p]),
    "dagr_compact_events": (C.c_int, [Dev, i64, Dev, Dev, Dev, Dev, C.c_int, C.c_int, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, p]),
    "dagr_ingest_events": (C.c_int, [Dev, Dev, Dev, Dev, i64, C.c_int, C.c_int, C.c_int, C.c_int, i64, C.c_int, Dev, Dev, Dev, Dev, Dev,
                                     Dev, Dev, Dev, p]),
    "dagr_window_bounds": (C.c_int, [Dev, i64, Dev, Dev, i64, Dev, Dev, p]),
    "dagr_window_gather": (C.c_int, [Dev, Dev, Dev, Dev, i64, Dev, Dev, C.c_int, i64, C.c_int, i64, Dev, Dev, Dev, Dev, p]),
    "dagr_stream_ingest": (C.c_int, [Dev, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev, C.c_int, p]),
    "dagr_frame_preprocess": (C.c_int, [Dev, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev, Dev, p]),
    "dagr_denormalize_pos": (C.c_int, [Dev, i64, C.c_int, C.c_int, C.c_int, Dev, p]),
    "dagr_prepare_events": (C.c_int, [Dev, Dev, Dev, C.c_int, i64, C.c_int, C.c_int, C.c_int, Dev, Dev, Dev, p]),
    "dagr_graph_sort": (C.c_int, [C.POINTER(Geom), Dev, Dev, Dev, i64, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, p]),
    "dagr_graph_sort_ring": (C.c_int, [C.POINTER(Geom), Dev, Dev, Dev, i64, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, p]),
    "dagr_stream_push": (C.c_int, [Dev, Dev, Dev, Dev, Dev, i64, C.c_int, C.c_int, p]),
    "dagr_stream_push_multi": (C.c_int, [Dev, Dev, Dev, Dev, Dev, i64, C.c_int, C.c_int, p]),
    "dagr_graph_sort_rings": (C.c_int, [C.POINTER(Geom), Dev, Dev, Dev, i64, C.c_int, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev,
                                        Dev, Dev, p]),
    "dagr_l1_build": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, C.POINTER(L1AParams), Dev, C.c_int, Dev, Dev, Dev, Dev, Dev,
                                Dev, C.c_int, p]),
    "dagr_l1a_tc_weights": (C.c_int, [C.POINTER(L1AParams), Host]),
    "dagr_l1_build_tc": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, C.POINTER(L1AParams), Dev, Dev, C.c_int, Dev, Dev, Dev,
                                   Dev, Dev, Dev, C.c_int, p]),
    "dagr_xa_permute": (C.c_int, [i64, Dev, C.c_int, Dev, Dev, C.c_int, p]),
    "dagr_l1_x0_image": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, C.c_int, C.c_int, Dev, p]),
    "dagr_l1_x0_image_live": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, C.c_int, C.c_int, Dev, p]),
    "dagr_l1_x0_image_planes": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, Dev, C.c_int, Dev, p]),
    "dagr_voxel_sample_max": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, Dev, C.c_int,
                                        C.c_int, C.c_int, p]),
    "dagr_voxel_sample_max_planes": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev, C.c_int,
                                               Dev, C.c_int, C.c_int, C.c_int, p]),
    "dagr_graph_export": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, i64, p]),
    "dagr_l1_tc_weights": (C.c_int, [Host, Host, C.c_int, Host]),
    "dagr_l1_conv_b_pool_voxel_tc": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, Dev, Dev, Dev, C.POINTER(L1BParams), Dev, Dev,
                                               C.c_int, Dev, Dev, Dev, Dev, Dev, Dev, Dev, C.c_int, Dev, Dev, C.c_int, p]),
    "dagr_l1_conv_a_image_tc": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, Dev, Dev, C.POINTER(L1ImgParams), Dev, Dev, Dev,
                                          Dev, Dev, C.c_int, p]),
    "dagr_l1_conv_a_image_inc": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, Dev, Dev, Dev, C.POINTER(L1ImgParams), Dev,
                                           C.c_int, Dev, Dev, Dev, Dev, C.c_int, p]),
    "dagr_voxel_sample_max_inc": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev,
                                            C.c_int, C.c_int, C.c_int, p]),
    "dagr_grid_cat_pos": (C.c_int, [C.POINTER(Grid), Dev, Dev, Dev, C.c_int, Dev, p]),
    "dagr_grid_conv": (C.c_int, [C.POINTER(Grid), Dev, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, Dev, Dev, Dev, Dev, Dev, Dev, C.c_int,
                                 f32, f32, Dev, p]),
    "dagr_grid_conv_last_instance": (C.c_int, []),
    "dagr_grid_linear_bn": (C.c_int, [i64, Dev, Dev, C.c_int, C.c_int, Dev, Dev, Dev, Dev, p]),
    "dagr_grid_pool": (C.c_int, [C.POINTER(Grid), C.POINTER(Grid), Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, C.c_int, C.c_int, Dev, Dev,
                                 Dev, Dev, Dev, Dev, Dev, p]),
    "dagr_grid_pool_finalize": (C.c_int, [C.POINTER(Grid), C.c_int, C.c_int, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, Dev, p]),
    "dagr_grid_temporal_filter": (C.c_int, [C.POINTER(Grid), Dev, Dev, Dev, p]),
    "dagr_grid_to_dense": (C.c_int, [C.POINTER(Grid), Dev, Dev, C.c_int, C.c_int, Dev, Dev, p]),
    "dagr_head_finish": (C.c_int, [C.POINTER(Grid), Dev, Dev, C.c_int, Dev, C.c_int, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int,
                                   C.c_int, Dev, p]),
    "dagr_head_finish_planes": (C.c_int, [C.POINTER(Grid), Dev, Dev, C.c_int, Dev, C.c_int, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int,
                                          C.c_int, C.c_int, Dev, C.c_int, Dev, p]),
    "dagr_postprocess_nms": (C.c_int, [Dev, C.c_int, C.c_int, C.c_int, f32, f32, C.c_int, C.c_int, C.c_int, Dev, Dev, p]),
    "dagr_sample_features": (C.c_int, [Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev, Dev, i64, C.c_int, C.c_int, Dev,
                                       C.c_int, C.c_int, p]),
    "dagr_sample_features_planes": (C.c_int, [Dev, C.c_int, Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev, Dev, i64, C.c_int,
                                              C.c_int, Dev, C.c_int, C.c_int, p]),
    # bf16 NHWC forms of the image-sampling calls (map as const void *, with its C)
    "dagr_l1_x0_image_bf16": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, Dev, p]),
    "dagr_l1_x0_image_live_bf16": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, Dev, p]),
    "dagr_l1_x0_image_planes_bf16": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev,
                                               C.c_int, Dev, p]),
    "dagr_voxel_sample_max_bf16": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, Dev, C.c_int,
                                             C.c_int, C.c_int, p]),
    "dagr_voxel_sample_max_inc_bf16": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev,
                                                 C.c_int, C.c_int, C.c_int, p]),
    "dagr_voxel_sample_max_planes_bf16": (C.c_int, [C.POINTER(Geom), i64, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev,
                                                    C.c_int, Dev, C.c_int, C.c_int, C.c_int, p]),
    "dagr_sample_features_bf16": (C.c_int, [Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev, Dev, i64, C.c_int, C.c_int, Dev,
                                            C.c_int, C.c_int, p]),
    "dagr_sample_features_planes_bf16": (C.c_int, [Dev, C.c_int, Dev, C.c_int, C.c_int, C.c_int, C.c_int, Dev, Dev, Dev, i64, C.c_int,
                                                   C.c_int, Dev, C.c_int, C.c_int, p]),
    "dagr_masked_lin": (C.c_int, [Dev, i64, Dev, Dev, Dev, Dev, C.c_int, C.c_int, C.c_int, p]),
    "dagr_masked_inplace_bn": (C.c_int, [Dev, i64, Dev, Dev, Dev, Dev, Dev, Dev, C.c_int, f32, p]),
    "dagr_masked_isdiff": (C.c_int, [Dev, i64, Dev, Dev, C.c_int, f32, f32, p]),
    "dagr_eval_workspace_bytes": (C.c_int, [i64, C.c_int, i64, i64, C.POINTER(i64)]),
    "dagr_evaluate_bbox": (C.c_int, [Dev, Dev, Dev, Dev, Dev, Dev, Dev, i64, C.c_int, i64, i64, C.POINTER(EvalParams), Dev, i64,
                                     Dev, Dev, p]),
    "dagr_interframe_targets_workspace_bytes": (C.c_int, [i64, i64, C.POINTER(i64)]),
    "dagr_interframe_targets": (C.c_int, [Dev, Dev, Dev, Dev, Dev, i64, i64, Dev, Dev, Dev, i64, C.c_int, C.c_int, C.c_int, f32, f32,
                                          i64, Dev, i64, Dev, Dev, Dev, p]),
    "dagr_eval_pack_workspace_bytes": (C.c_int, [i64, C.POINTER(i64)]),
    "dagr_eval_pack_detections": (C.c_int, [Dev, Dev, i64, C.c_int, Dev, Dev, C.c_int, Dev, i64, Dev, Dev, Dev, Dev, p]),
}

EXPORTS = tuple(_SIGS.keys())


def lib_path() -> Path:
    return _LIB_PATH


def _entry(name, fn):
    """fn, with an argument its type refuses raised as RuntimeError naming the entry point and the argument (ctypes
    reports it as ArgumentError); nothing is launched."""
    def call(*args):
        try:
            return fn(*args)
        except C.ArgumentError as e:
            raise RuntimeError(f"dagr_b200: {name} {e}") from None
    call.__name__ = name
    return call


def load():
    """Load (building in-tree with nvcc if needed) and return the ctypes handle."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.environ.get("DAGR_B200_LIB"):
        from . import build as _build
        if _build.needs_build():                          # missing, or built from other sources than the ones in the tree
            try:
                _build.build(force=True)
            except Exception as e:
                if not _LIB_PATH.exists():
                    raise RuntimeError(f"dagr_b200: could not build the CUDA extension: {e}") from e
                import warnings
                warnings.warn(f"dagr_b200: libdagr_b200.so is older than its sources and could not be rebuilt ({e})")
    if not _LIB_PATH.exists():
        raise RuntimeError(f"dagr_b200: CUDA extension {_LIB_PATH} is missing and could not be built; "
                           "there is no CPU fallback")
    lib = C.CDLL(str(_LIB_PATH))
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
        setattr(lib, name, _entry(name, fn))
    if lib.dagr_abi_version() != 3:
        raise RuntimeError("dagr_b200: ABI version mismatch between python host and libdagr_b200.so")
    _lib = lib
    return lib


def check(code: int, what: str = ""):
    if code != 0:
        msg = load().dagr_last_error()
        raise RuntimeError(f"dagr_b200 {what} failed ({code}): {msg.decode() if msg else ''}")


def ptr(t):
    """raw address of a tensor (None -> NULL), for tests and tools that work with addresses; product code passes the
    tensor itself (Dev)."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"dagr_b200: `{name}` must be a CUDA tensor (no CPU fallback on the product path)")
    if not t.is_contiguous():
        raise RuntimeError(f"dagr_b200: `{name}` must be contiguous")
