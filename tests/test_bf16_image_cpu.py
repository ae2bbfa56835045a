"""bf16 image branch without a GPU: the eight _bf16 sampling entry points are exported and declared, their argument checks
refuse bad input with DAGR_E_ARG and a message naming the entry point before anything is launched, and DAGR.image_precision
takes only "tf32" / "bf16" and never touches the model's own fp32 weights."""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

from tests.helpers import make_model

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first
ROOT = Path(__file__).resolve().parent.parent
NAMES = ["dagr_l1_x0_image_bf16", "dagr_l1_x0_image_live_bf16", "dagr_l1_x0_image_planes_bf16", "dagr_voxel_sample_max_bf16",
         "dagr_voxel_sample_max_inc_bf16", "dagr_voxel_sample_max_planes_bf16", "dagr_sample_features_bf16",
         "dagr_sample_features_planes_bf16"]


def test_bf16_entry_points_are_exported_declared_and_counted():
    from dagr_b200 import _lib
    from dagr_b200.engine import Engine
    lib = _lib.load()
    header = (ROOT / "include" / "dagr_b200.h").read_text()
    for n in NAMES:
        assert n in _lib.EXPORTS
        getattr(lib, n)
        assert re.search(rf"\bint {n}\(", header), n
        assert Engine._NKERNELS[n] == 1
        # the fp32 form keeps its signature and ABI: same argument count, plus C for the x0 forms
        fp32 = n[: -len("_bf16")]
        extra = 1 if "x0_image" in n else 0
        assert len(_lib._SIGS[n][1]) == len(_lib._SIGS[fp32][1]) + extra
    assert lib.dagr_abi_version() == 2


def _geom(B=2):
    from dagr_b200.geometry import Geometry
    return Geometry(240, 180, B, device="cpu")


def _x0(lib, a, N=1 << 10, nplanes=4, stride=4, C=16):
    return lib.dagr_l1_x0_image_bf16(a["g"], N, a["xyb"], None, a["img"], C, 8, 8, a["out"], None)


def _x0_live(lib, a, N=1 << 10, nplanes=4, stride=4, C=16):
    return lib.dagr_l1_x0_image_live_bf16(a["g"], N, a["start"], a["xyb"], None, a["img"], C, 8, 8, a["out"], None)


def _x0_planes(lib, a, N=1 << 10, nplanes=4, stride=4, C=16):
    return lib.dagr_l1_x0_image_planes_bf16(a["g"], N, a["start"], a["xyb"], None, a["img"], C, 8, 8, nplanes, a["plane"], stride,
                                            a["out"], None)


def _vox(lib, a, N=1 << 10, nplanes=4, stride=4, C=64):
    return lib.dagr_voxel_sample_max_bf16(a["g"], N, a["start"], a["xyb"], a["img"], C, 8, 8, a["out"], 80, 16, 0, None)


def _vox_inc(lib, a, N=1 << 10, nplanes=4, stride=4, C=64):
    return lib.dagr_voxel_sample_max_inc_bf16(a["g"], N, a["start"], a["xyb"], a["ti"], a["img"], C, 8, 8, 0, a["persist"], a["out"],
                                              80, 16, 0, None)


def _vox_planes(lib, a, N=1 << 10, nplanes=4, stride=4, C=64):
    return lib.dagr_voxel_sample_max_planes_bf16(a["g"], N, a["start"], a["xyb"], a["img"], C, 8, 8, nplanes, a["plane"], stride,
                                                 a["out"], 80, 16, 0, None)


def _sample(lib, a, N=1 << 10, nplanes=4, stride=4, C=64):
    return lib.dagr_sample_features_bf16(a["img"], 2, C, 8, 8, a["posx"], a["posy"], a["bidx"], N, 240, 180, a["out"], 80, 16, None)


def _sample_planes(lib, a, N=1 << 10, nplanes=4, stride=4, C=64):
    return lib.dagr_sample_features_planes_bf16(a["img"], nplanes, a["plane"], stride, C, 8, 8, a["posx"], a["posy"], a["bidx"], N,
                                                240, 180, a["out"], 80, 16, None)


ENTRY = dict(dagr_l1_x0_image_bf16=(_x0, ["g", "xyb", "img", "out"]),
             dagr_l1_x0_image_live_bf16=(_x0_live, ["g", "start", "xyb", "img", "out"]),
             dagr_l1_x0_image_planes_bf16=(_x0_planes, ["g", "start", "xyb", "img", "plane", "out"]),
             dagr_voxel_sample_max_bf16=(_vox, ["g", "start", "xyb", "img", "out"]),
             dagr_voxel_sample_max_inc_bf16=(_vox_inc, ["g", "start", "xyb", "ti", "img", "persist", "out"]),
             dagr_voxel_sample_max_planes_bf16=(_vox_planes, ["g", "start", "xyb", "img", "plane", "out"]),
             dagr_sample_features_bf16=(_sample, ["img", "posx", "posy", "bidx", "out"]),
             dagr_sample_features_planes_bf16=(_sample_planes, ["img", "plane", "posx", "posy", "bidx", "out"]))
PLANES = sorted(n for n in ENTRY if "planes" in n)


def _args(geom):
    a = {k: BAD for k in ("start", "xyb", "ti", "img", "plane", "out", "persist", "posx", "posy", "bidx")}
    a["g"] = C.byref(geom.c_geom)
    return a


def test_entry_table_covers_every_bf16_entry_point():
    assert sorted(ENTRY) == sorted(NAMES)


@pytest.mark.parametrize("name,null", [(n, p) for n, (_, ps) in ENTRY.items() for p in ps])
def test_bf16_entry_points_reject_null_pointers(name, null):
    from dagr_b200 import _lib
    lib = _lib.load()
    call, _ = ENTRY[name]
    a = _args(_geom())
    a[null] = None
    assert call(lib, a) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert name in msg and "null" in msg, msg


@pytest.mark.parametrize("name,kw,needle", [(n, kw, "N out of range") for n in sorted(ENTRY) for kw in (dict(N=-1), dict(N=1 << 31))]
                         + [(n, kw, m) for n in PLANES for kw, m in ((dict(nplanes=0), "nplanes"), (dict(nplanes=-3), "nplanes"),
                                                                    (dict(stride=0), "plane_stride"))])
def test_bf16_entry_points_reject_bad_counts(name, kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    call, _ = ENTRY[name]
    assert call(lib, _args(_geom()), **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert name in msg and needle in msg, msg


@pytest.mark.parametrize("name", [n for n in NAMES if "x0_image" in n])
def test_bf16_x0_forms_take_only_the_16_channel_tap(name):
    from dagr_b200 import _lib
    lib = _lib.load()
    for C_ in (8, 64):
        assert ENTRY[name][0](lib, _args(_geom()), C=C_) == E_ARG
        assert "16" in lib.dagr_last_error().decode()


@pytest.mark.parametrize("name", [n for n in NAMES if "voxel" in n])
def test_bf16_voxel_forms_reject_channels_past_the_row(name):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert ENTRY[name][0](lib, _args(_geom()), C=65) == E_ARG           # c0 = 16, ldx = 80
    assert "ldx" in lib.dagr_last_error().decode()


def test_bf16_voxel_inc_refuses_mean_pooling():
    from dagr_b200 import _lib
    lib = _lib.load()
    a = _args(_geom())
    assert lib.dagr_voxel_sample_max_inc_bf16(a["g"], 1 << 10, BAD, BAD, BAD, BAD, 64, 8, 8, 0, BAD, BAD, 80, 16, 1, None) == E_ARG
    assert "pool_mean" in lib.dagr_last_error().decode()
    assert lib.dagr_voxel_sample_max_inc_bf16(a["g"], 1 << 10, BAD, BAD, BAD, BAD, 64, 8, 8, -1, BAD, BAD, 80, 16, 0, None) == E_ARG
    assert "min_idx" in lib.dagr_last_error().decode()


def test_image_precision_takes_tf32_or_bf16_only():
    model, _ = make_model("n", 180, 240, use_image=True, img_net="resnet18")
    assert model.image_precision == "tf32"
    for bad in ("fp16", "BF16", "fp32", None, 16):
        with pytest.raises(ValueError, match="image_precision"):
            model.image_precision = bad
        assert model.image_precision == "tf32"
    model.image_precision = "bf16"
    assert model.image_precision == "bf16"
    assert "image_precision" not in vars(model.args)                   # a model attribute, not an argparse / yaml key
    from dagr_b200.model.image_branch import ImageBranch
    with pytest.raises(ValueError, match="image precision"):
        ImageBranch(model).run(torch.zeros(1, 3, 180, 240), precision="fp16")


def test_switching_precision_leaves_the_fp32_state_dict_bit_identical():
    import copy
    model, _ = make_model("n", 180, 240, use_image=True, img_net="resnet18")
    before = {k: v.clone() for k, v in model.state_dict().items()}
    model.image_precision = "bf16"
    from dagr_b200.model.image_branch import _bf16_copy
    net = _bf16_copy(model.backbone.net)                               # the branch's own copy: the model's modules stay fp32
    assert any(p.dtype == torch.bfloat16 for p in net.parameters())
    model.image_precision = "tf32"
    after = model.state_dict()
    assert before.keys() == after.keys()
    for k, v in before.items():
        assert after[k].dtype == v.dtype and torch.equal(after[k], v), k
        assert after[k].is_contiguous(), k
    assert copy.deepcopy(model).image_precision == "tf32"
