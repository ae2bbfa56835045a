"""The ctypes binding's pointer argument types (no GPU): device pointers take CUDA tensors and refuse host memory before any
launch, *_host pointers refuse CUDA tensors, and every declaration of include/dagr_b200.h is bound argument by argument."""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

from dagr_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent

# argument count of every entry point: the C-ABI (DAGR_ABI_VERSION 3) is bound unchanged
ARG_COUNTS = {
    "dagr_abi_version": 0, "dagr_last_error": 0, "dagr_scan_blocks": 1, "dagr_check_config": 5, "dagr_event_workspace_bytes": 3,
    "dagr_pool_workspace_bytes": 3, "dagr_downsample_events": 17, "dagr_compact_events": 17, "dagr_ingest_events": 20,
    "dagr_window_bounds": 8, "dagr_window_gather": 16, "dagr_stream_ingest": 12, "dagr_frame_preprocess": 11,
    "dagr_denormalize_pos": 7, "dagr_prepare_events": 12, "dagr_graph_sort": 16, "dagr_graph_sort_ring": 17, "dagr_stream_push": 9,
    "dagr_stream_push_multi": 9, "dagr_graph_sort_rings": 18, "dagr_l1_build": 17, "dagr_l1a_tc_weights": 2, "dagr_l1_build_tc": 18,
    "dagr_xa_permute": 7, "dagr_l1_x0_image": 9, "dagr_l1_x0_image_live": 10, "dagr_l1_x0_image_planes": 13,
    "dagr_voxel_sample_max": 13, "dagr_voxel_sample_max_planes": 16, "dagr_graph_export": 12, "dagr_l1_tc_weights": 4,
    "dagr_l1_conv_b_pool_voxel_tc": 25, "dagr_l1_conv_a_image_tc": 16, "dagr_l1_conv_a_image_inc": 18,
    "dagr_voxel_sample_max_inc": 16, "dagr_grid_cat_pos": 7, "dagr_grid_conv": 19, "dagr_grid_conv_last_instance": 0,
    "dagr_grid_linear_bn": 10, "dagr_grid_pool": 20, "dagr_grid_pool_finalize": 13, "dagr_grid_temporal_filter": 5,
    "dagr_grid_to_dense": 8, "dagr_head_finish": 15, "dagr_head_finish_planes": 18, "dagr_postprocess_nms": 12,
    "dagr_sample_features": 15, "dagr_sample_features_planes": 17, "dagr_l1_x0_image_bf16": 10, "dagr_l1_x0_image_live_bf16": 11,
    "dagr_l1_x0_image_planes_bf16": 14, "dagr_voxel_sample_max_bf16": 13, "dagr_voxel_sample_max_inc_bf16": 16,
    "dagr_voxel_sample_max_planes_bf16": 16, "dagr_sample_features_bf16": 15, "dagr_sample_features_planes_bf16": 17,
    "dagr_masked_lin": 10, "dagr_masked_inplace_bn": 11, "dagr_masked_isdiff": 8, "dagr_eval_workspace_bytes": 5,
    "dagr_evaluate_bbox": 17, "dagr_interframe_targets_workspace_bytes": 3, "dagr_interframe_targets": 23,
    "dagr_eval_pack_workspace_bytes": 2, "dagr_eval_pack_detections": 14,
}


def _declarations():
    """name -> parameter declarations of every function in include/dagr_b200.h (comments removed)."""
    src = re.sub(r"/\*.*?\*/", " ", (ROOT / "include" / "dagr_b200.h").read_text(), flags=re.S)
    decls = {}
    for m in re.finditer(r"^[A-Za-z_][\w *]*?\b(dagr_\w+)\s*\(([^)]*)\)\s*;", src, flags=re.M):
        params = m.group(2).strip()
        decls[m.group(1)] = [] if params in ("", "void") else [" ".join(a.split()) for a in params.split(",")]
    return decls


def _pointer_kind(fn, param):
    """how the binding must declare a parameter: None for a scalar, else stream / struct / string / out / host / dev."""
    if "*" not in param:
        return None
    name = re.findall(r"\w+", param)[-1]
    if name == "stream":
        return "stream"
    if re.search(r"\b(struct\s+)?dagr_\w+", param.split("*")[0]):
        return "struct"
    if re.match(r"(const )?char \*", param):
        return "string"
    if fn.endswith("_workspace_bytes"):
        return "out"
    return "host" if name.endswith("_host") else "dev"


def test_every_declaration_is_bound_with_its_pointer_types():
    decls = _declarations()
    assert set(decls) == set(_lib._SIGS) == set(ARG_COUNTS)
    kinds = set()
    for fn, params in decls.items():
        args = _lib._SIGS[fn][1]
        assert len(args) == len(params) == ARG_COUNTS[fn], fn
        for i, (param, a) in enumerate(zip(params, args)):
            kind = _pointer_kind(fn, param)
            kinds.add(kind)
            where = f"{fn} argument {i + 1} ({param})"
            if kind == "dev":
                assert a is _lib.Dev, where
            elif kind == "host":
                assert a is _lib.Host, where
            elif kind == "stream":
                assert a is C.c_void_p, where
            elif kind in ("struct", "out"):
                assert issubclass(a, C._Pointer), where
            elif kind == "string":
                assert a is C.c_char_p, where
            else:
                assert a not in (_lib.Dev, _lib.Host, C.c_void_p), where
    assert kinds == {None, "dev", "host", "stream", "struct", "out", "string"}
    host = [(fn, p) for fn, params in decls.items() for p in params if _pointer_kind(fn, p) == "host"]
    assert sorted(fn for fn, _ in host) == ["dagr_l1_tc_weights"] * 3 + ["dagr_l1a_tc_weights"]


def test_dev_passes_raw_addresses_and_refuses_host_tensors():
    def address(obj):
        return C.cast(_lib.Dev.from_param(obj), C.c_void_p).value
    assert address(None) is None
    assert address(0x7F0012345678) == 0x7F0012345678                 # a full 64-bit address, not cut to a C int
    assert address(C.c_void_p(0x1000)) == 0x1000
    for t in (torch.zeros(4), torch.zeros(4, dtype=torch.int32)[1:]):
        with pytest.raises(RuntimeError, match="cpu tensor where the library takes a device pointer"):
            _lib.Dev.from_param(t)


def test_host_takes_ctypes_buffers_and_refuses_cuda_tensors():
    class CudaLike:
        is_cuda = True
    with pytest.raises(RuntimeError, match="host pointer"):
        _lib.Host.from_param(CudaLike())
    buf = (C.c_float * 4)()
    assert _lib.Host.from_param(buf) is not None


def test_entry_point_refuses_a_host_tensor_before_the_call():
    """a CPU tensor for a device pointer: RuntimeError naming the entry point and the argument; the C function is never
    entered, so the library's last error is untouched."""
    lib = _lib.load()
    assert lib.dagr_masked_lin(None, -1, None, None, None, None, 4, 5, 0, None) == -1    # refused by the library: K < 0
    before = lib.dagr_last_error()
    assert b"K < 0" in before                  # the call below, if entered, would replace it with its null-pointer message
    x = torch.zeros((3, 4))
    with pytest.raises(RuntimeError, match=r"dagr_masked_lin argument 3: .*cpu tensor where the library takes a device pointer"):
        lib.dagr_masked_lin(None, 1, x, None, None, None, 4, 5, 0, None)
    assert lib.dagr_last_error() == before
    assert lib.dagr_masked_lin.__name__ == "dagr_masked_lin"
