"""tests/shipped_shapes.py, the coarse-level shapes of the shipped configurations, checked without a GPU: it is
deterministic, it reads the models the way the engine does, and it holds the shapes the kernel-level tests once missed."""
import torch

from tests import shipped_shapes as S


def test_shipped_shapes_configurations():
    """every config/*.yaml (size, dataset) plus dagr-n on N-Caltech101, image fusion off and on"""
    assert set(S.configs()) == {(s, d, i) for s, d in (("n", "dsec"), ("s", "dsec"), ("m", "dsec"), ("l", "dsec"),
                                                       ("l", "ncaltech101"), ("n", "ncaltech101")) for i in (False, True)}


def test_shipped_shapes_are_deterministic():
    """a second, independent build of every model gives the same launches"""
    from dagr_b200.model.dagr import DAGR
    for cfg in S.configs():
        W, H = S.SENSOR[cfg[1]]
        torch.manual_seed(123)
        again = S.launches_of(DAGR(S.config_args(*cfg), height=H, width=W).eval())
        assert again == S.launches(*cfg), cfg
    assert S.shipped() == S.shipped.__wrapped__()


def test_shipped_shapes_follow_the_layer_inputs():
    """each pooled width is what the next layer reads: its conv_block1 input minus the two position channels (so the
    workspace rule C_lv + image taps agrees with the module tree), and cat_pos appends to the same widths"""
    from dagr_b200.model.dagr import DAGR
    for cfg in S.configs():
        W, H = S.SENSOR[cfg[1]]
        model = DAGR(S.config_args(*cfg), height=H, width=W).eval()
        bb = model.backbone
        ins = [getattr(bb, n).conv_block1.conv.in_channels - 2 for n in ("layer2", "layer3", "layer4", "layer5")]
        L = S.launches(*cfg)
        assert {w for w, _ in L["pool"]} == set(ins[1:]), cfg
        assert L["cat_pos"] == sorted(set(ins)), cfg
        assert ("mean" in {a for _, a in L["pool"]}) and len(L["pool"]) <= 3
        assert {(ci, co) for ci, co in L["linear_bn"]} == {(i + 2, getattr(bb, n).conv_block2.conv.out_channels)
                                                           for i, n in zip(ins, ("layer2", "layer3", "layer4", "layer5"))}


def test_shipped_shapes_hold_the_shapes_once_untested():
    sh = S.shipped()
    conv = {(ci, co) for ci, co, _, _ in sh["conv"]}
    blocks = {(ci, co, off, ld) for ci, co, off, ld in sh["conv"] if ld != ci}
    dense = {(66, 32), (34, 32), (32, 32), (32, 64), (64, 128), (66, 96), (98, 96), (96, 96), (128, 128),       # events
             (82, 64), (98, 32), (130, 64), (162, 96), (194, 96), (194, 128), (258, 128)}                    # fusion
    assert dense <= conv
    for C in (32, 64, 96, 128):                # cls_pred on the first half, reg_pred | obj_pred on the second
        assert {(C, 2, 0, 2 * C), (C, 5, C, 2 * C)} <= blocks, C
    assert {(32, 100, 0, 64), (128, 100, 0, 256)} <= blocks
    assert {w for w, _ in sh["pool"]} == {32, 64, 96, 128, 160, 192, 256}
    assert {(w, "mean") for w in (32, 64, 96, 128, 192, 256)} <= set(sh["pool"])
    assert {(34, 32), (66, 32), (98, 96), (66, 96), (130, 128)} <= set(sh["linear_bn"])
    assert sh["head_finish"] == [(2, False), (2, True), (100, False), (100, True)]
    assert {(2, 2, 0), (100, 100, 0), (4, 5, 0), (1, 5, 4)} == {t[:3] for t in sh["to_dense"]}
    assert 16 in sh["cat_pos"] and 80 in sh["cat_pos"]


def test_shipped_shapes_conv_labels():
    """the engine's profile labels of dagr-n on DSEC, written out"""
    assert S.conv_labels("n", "dsec", False) == [
        "grid_conv_L1_18x64", "grid_conv_L1_64x64", "grid_conv_L2_32x32", "grid_conv_L2_66x32", "grid_conv_L3_32x2",
        "grid_conv_L3_32x32", "grid_conv_L3_32x5", "grid_conv_L3_32x64", "grid_conv_L3_34x32", "grid_conv_L4_32x2",
        "grid_conv_L4_32x32", "grid_conv_L4_32x5", "grid_conv_L4_32x64", "grid_conv_L4_34x32"]
