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
    "dagr_downsample_events": (C.c_int, [p, p, p, i64, C.c_int, C.c_int, C.c_int, C.c_int, p, p, p, p, p, p, p, p, p]),
    "dagr_compact_events": (C.c_int, [p, i64, p, p, p, p, C.c_int, C.c_int, p, p, p, p, p, p, p, p, p]),
    "dagr_ingest_events": (C.c_int, [p, p, p, p, i64, C.c_int, C.c_int, C.c_int, C.c_int, i64, C.c_int, p, p, p, p, p, p, p, p, p]),
    "dagr_stream_ingest": (C.c_int, [p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, p, p, C.c_int, p]),
    "dagr_frame_preprocess": (C.c_int, [p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, p, p, p, p]),
    "dagr_denormalize_pos": (C.c_int, [p, i64, C.c_int, C.c_int, C.c_int, p, p]),
    "dagr_prepare_events": (C.c_int, [p, p, p, C.c_int, i64, C.c_int, C.c_int, C.c_int, p, p, p, p]),
    "dagr_graph_sort": (C.c_int, [C.POINTER(Geom), p, p, p, i64, p, p, p, p, p, p, p, p, p, p, p]),
    "dagr_graph_sort_ring": (C.c_int, [C.POINTER(Geom), p, p, p, i64, p, p, p, p, p, p, p, p, p, p, p, p]),
    "dagr_stream_push": (C.c_int, [p, p, p, p, p, i64, C.c_int, C.c_int, p]),
    "dagr_stream_push_multi": (C.c_int, [p, p, p, p, p, i64, C.c_int, C.c_int, p]),
    "dagr_graph_sort_rings": (C.c_int, [C.POINTER(Geom), p, p, p, i64, C.c_int, p, p, p, p, p, p, p, p, p, p, p, p]),
    "dagr_graph_search": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, p, p]),
    "dagr_l1_build": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, C.POINTER(L1AParams), p, C.c_int, p, p, p, p, p, p, C.c_int, p]),
    "dagr_l1a_tc_weights": (C.c_int, [C.POINTER(L1AParams), p]),
    "dagr_l1_build_tc": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, C.POINTER(L1AParams), p, p, C.c_int, p, p, p, p, p, p, C.c_int, p]),
    "dagr_xa_permute": (C.c_int, [i64, p, C.c_int, p, p, C.c_int, p]),
    "dagr_l1_x0_image": (C.c_int, [C.POINTER(Geom), i64, p, p, p, C.c_int, C.c_int, p, p]),
    "dagr_l1_x0_image_live": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, C.c_int, C.c_int, p, p]),
    "dagr_l1_x0_image_planes": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, C.c_int, C.c_int, C.c_int, p, C.c_int, p, p]),
    "dagr_l1_conv_a_image": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, p, C.POINTER(L1ImgParams), p, p, p, p, C.c_int, p]),
    "dagr_voxel_sample_max": (C.c_int, [C.POINTER(Geom), i64, p, p, p, C.c_int, C.c_int, C.c_int, p, C.c_int, C.c_int, C.c_int, p]),
    "dagr_voxel_sample_max_planes": (C.c_int, [C.POINTER(Geom), i64, p, p, p, C.c_int, C.c_int, C.c_int, C.c_int, p, C.c_int, p, C.c_int,
                                               C.c_int, C.c_int, p]),
    "dagr_graph_export": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, p, p, p, i64, p]),
    "dagr_l1_conv_a": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, C.POINTER(L1AParams), p, p]),
    "dagr_l1_conv_b_pool": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, p, C.POINTER(L1BParams), p, p, p]),
    "dagr_l1_conv_b_pool_voxel": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, p, p, p, C.POINTER(L1BParams), p, C.c_int, p, p, p, p, p, p, p, C.c_int, p, p, C.c_int, p]),
    "dagr_l1_tc_weights": (C.c_int, [p, p, C.c_int, p]),
    "dagr_l1_conv_b_pool_voxel_tc": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, p, p, C.POINTER(L1BParams), p, p, C.c_int, p, p, p, p, p, p, p, C.c_int, p, p, C.c_int, p]),
    "dagr_l1_conv_a_image_tc": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, p, C.POINTER(L1ImgParams), p, p, p, p, p, C.c_int, p]),
    "dagr_l1_conv_a_image_inc": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, p, p, p, C.POINTER(L1ImgParams), p, C.c_int, p, p, p, p,
                                           C.c_int, p]),
    "dagr_voxel_sample_max_inc": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, C.c_int, C.c_int, C.c_int, C.c_int, p, p, C.c_int, C.c_int,
                                            C.c_int, p]),
    "dagr_pool1_finalize": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, C.c_int, p, p, p, p, p, p]),
    "dagr_grid_cat_pos": (C.c_int, [C.POINTER(Grid), p, p, p, C.c_int, p, p]),
    "dagr_grid_conv": (C.c_int, [C.POINTER(Grid), p, p, p, p, C.c_int, C.c_int, C.c_int, p, p, p, p, p, p, C.c_int, f32, f32, p, p]),
    "dagr_grid_linear_bn": (C.c_int, [i64, p, p, C.c_int, C.c_int, p, p, p, p, p]),
    "dagr_grid_pool": (C.c_int, [C.POINTER(Grid), C.POINTER(Grid), p, p, p, p, p, p, p, p, C.c_int, C.c_int,
                                 p, p, p, p, p, p, p, p]),
    "dagr_grid_pool_finalize": (C.c_int, [C.POINTER(Grid), C.c_int, C.c_int, p, p, p, p, p, p, p, p, p, p]),
    "dagr_grid_temporal_filter": (C.c_int, [C.POINTER(Grid), p, p, p, p]),
    "dagr_grid_to_dense": (C.c_int, [C.POINTER(Grid), p, p, C.c_int, C.c_int, p, p, p]),
    "dagr_head_decode": (C.c_int, [p, p, p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, p, p]),
    "dagr_head_finish": (C.c_int, [C.POINTER(Grid), p, p, C.c_int, p, C.c_int, p, p, p, C.c_int, C.c_int, C.c_int, C.c_int, p, p]),
    "dagr_head_finish_planes": (C.c_int, [C.POINTER(Grid), p, p, C.c_int, p, C.c_int, p, p, p, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_int, p, C.c_int, p, p]),
    "dagr_postprocess_nms": (C.c_int, [p, C.c_int, C.c_int, C.c_int, f32, f32, C.c_int, C.c_int, C.c_int, p, p, p]),
    "dagr_sample_features": (C.c_int, [p, C.c_int, C.c_int, C.c_int, C.c_int, p, p, p, i64, C.c_int, C.c_int, p,
                                       C.c_int, C.c_int, p]),
    "dagr_sample_features_planes": (C.c_int, [p, C.c_int, p, C.c_int, C.c_int, C.c_int, C.c_int, p, p, p, i64, C.c_int, C.c_int, p,
                                              C.c_int, C.c_int, p]),
    # bf16 NHWC forms of the image-sampling calls (map as const void *, with its C)
    "dagr_l1_x0_image_bf16": (C.c_int, [C.POINTER(Geom), i64, p, p, p, C.c_int, C.c_int, C.c_int, p, p]),
    "dagr_l1_x0_image_live_bf16": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, C.c_int, C.c_int, C.c_int, p, p]),
    "dagr_l1_x0_image_planes_bf16": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, C.c_int, C.c_int, C.c_int, C.c_int, p, C.c_int, p, p]),
    "dagr_voxel_sample_max_bf16": (C.c_int, [C.POINTER(Geom), i64, p, p, p, C.c_int, C.c_int, C.c_int, p, C.c_int, C.c_int, C.c_int, p]),
    "dagr_voxel_sample_max_inc_bf16": (C.c_int, [C.POINTER(Geom), i64, p, p, p, p, C.c_int, C.c_int, C.c_int, C.c_int, p, p, C.c_int,
                                                 C.c_int, C.c_int, p]),
    "dagr_voxel_sample_max_planes_bf16": (C.c_int, [C.POINTER(Geom), i64, p, p, p, C.c_int, C.c_int, C.c_int, C.c_int, p, C.c_int, p,
                                                    C.c_int, C.c_int, C.c_int, p]),
    "dagr_sample_features_bf16": (C.c_int, [p, C.c_int, C.c_int, C.c_int, C.c_int, p, p, p, i64, C.c_int, C.c_int, p, C.c_int, C.c_int,
                                            p]),
    "dagr_sample_features_planes_bf16": (C.c_int, [p, C.c_int, p, C.c_int, C.c_int, C.c_int, C.c_int, p, p, p, i64, C.c_int, C.c_int,
                                                   p, C.c_int, C.c_int, p]),
    "dagr_masked_lin":(C.c_int, [p, i64, p, p, p, p, C.c_int, C.c_int, C.c_int, p]),
    "dagr_masked_inplace_bn": (C.c_int, [p, i64, p, p, p, p, p, p, C.c_int, f32, p]),
    "dagr_masked_isdiff": (C.c_int, [p, i64, p, p, C.c_int, f32, f32, p]),
}

EXPORTS = tuple(_SIGS.keys())


def lib_path() -> Path:
    return _LIB_PATH


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
    if lib.dagr_abi_version() != 2:
        raise RuntimeError("dagr_b200: ABI version mismatch between python host and libdagr_b200.so")
    _lib = lib
    return lib


def check(code: int, what: str = ""):
    if code != 0:
        msg = load().dagr_last_error()
        raise RuntimeError(f"dagr_b200 {what} failed ({code}): {msg.decode() if msg else ''}")


def ptr(t):
    """device pointer of a tensor (None -> NULL)."""
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
