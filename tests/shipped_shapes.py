"""The coarse-level launches of every shipped configuration, derived from the models themselves.

A configuration is one (size, dataset) with a config/*.yaml, plus dagr-n on N-Caltech101 (which the parity tests build),
each with use_image off and on.  For each, the model is built on the CPU and its module tree read the way Engine.pack and
Engine.forward_events read it:
  * dagr_grid_conv: (level, Cin, Cout, column offset, ldin) -- the two SplineConvs of layer2..5 and, per head scale, the
    stem, cls_conv | reg_conv as ONE C -> 2C launch, cls_pred on columns [0, C) and reg_pred | obj_pred as ONE C -> 5 launch
    on columns [C, 2C) of the [cells, 2C] output (ldin = 2C).  `level` is the 1-based grid level of the engine's
    grid_conv_L{level}_{Cin}x{Cout} profile labels; ldin = Cin for a dense input;
  * dagr_grid_linear_bn: (Cin, Cout) of each layer's skip branch;
  * dagr_grid_cat_pos: the width Cx of the features that get (x, y) appended in front of each layer;
  * dagr_grid_pool / _finalize: (pooled width, aggregation) of pool2..4 -- C_lv plus the image taps as Engine.workspace
    counts them, pool4 always mean (net.py:96-97);
  * dagr_head_finish: (nc, with CNN maps) per head scale;
  * dagr_grid_to_dense: (C, ldx, column offset, with CNN maps) of the dense cls, reg and obj maps.
tests/test_coarse_shapes_gpu.py runs each coarse kernel at these shapes and checks the conv set against the labels the
engine records; tests/test_shipped_shapes_cpu.py pins the derivation.
"""
import re
from functools import lru_cache
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
# sensor size of each dataset (DSEC after the 2x down-sizing, N-Caltech101); the shapes do not depend on it
SENSOR = dict(dsec=(640, 480), ncaltech101=(240, 180))
KINDS = ("conv", "linear_bn", "cat_pos", "pool", "head_finish", "to_dense")


def configs():
    """[(size, dataset, use_image)]: every config/dagr-<size>-*.yaml plus dagr-n on N-Caltech101, image fusion off and on"""
    import yaml
    out = set()
    for f in sorted((ROOT / "config").glob("dagr-*.yaml")):
        size = re.fullmatch(r"dagr-([nsml])-.*\.yaml", f.name).group(1)
        out.add((size, yaml.safe_load(f.read_text())["dataset"]))
    out.add(("n", "ncaltech101"))
    return [(s, d, img) for s, d in sorted(out) for img in (False, True)]


def config_args(size, dataset, use_image):
    """the argparse namespace of one configuration: the yaml's network keys where a yaml exists, the defaults otherwise"""
    import yaml
    from dagr_b200.utils.args import default_args
    over = {}
    for f in sorted((ROOT / "config").glob(f"dagr-{size}-*.yaml")):
        cfg = yaml.safe_load(f.read_text())
        if cfg["dataset"] == dataset:
            over = {k: v for k, v in cfg.items() if k not in ("task", "dataset", "batch_size")}
    return default_args(size, dataset=dataset, batch_size=2, **dict(over, use_image=use_image))


def launches_of(model):
    """{kind: sorted list of the launch tuples described in the module docstring} of one model"""
    bb, hd = model.backbone, model.head
    use_image = bool(bb.use_image)
    fc = list(bb.net.feature_channels) if use_image else []
    C_lv = list(bb.output_channels)                                   # [16, 64, C, C, C]
    res = {k: set() for k in KINDS}
    for lv, name in enumerate(("layer2", "layer3", "layer4", "layer5")):
        layer = getattr(bb, name)
        a, b = layer.conv_block1.conv, layer.conv_block2.conv
        res["conv"].add((lv + 1, a.in_channels, a.out_channels, 0, a.in_channels))
        res["conv"].add((lv + 1, b.in_channels, b.out_channels, 0, b.in_channels))
        wT = layer.conv_block2.lin.mlp.weight.t()
        res["linear_bn"].add(tuple(wT.shape))
        res["cat_pos"].add(a.in_channels - 2)
    for lv in (1, 2, 3):                                              # pool2..4 pool into grid level lv (0-based)
        aggr = "mean" if lv == 3 else model.args.pooling_aggr
        res["pool"].add((C_lv[lv] + (fc[lv + 1] if use_image else 0), aggr))
    nc = bb.num_classes
    levels = (3, 4) if hd.num_scales == 2 else (4,)
    for k, lv in enumerate(levels):
        sfx = str(k + 1)
        stem, cc, rc = (getattr(hd, n + sfx).conv for n in ("stem", "cls_conv", "reg_conv"))
        cp, rp, op = (getattr(hd, n + sfx) for n in ("cls_pred", "reg_pred", "obj_pred"))
        Cf = cc.out_channels
        res["conv"].add((lv, stem.in_channels, stem.out_channels, 0, stem.in_channels))
        res["conv"].add((lv, cc.in_channels, cc.out_channels + rc.out_channels, 0, cc.in_channels))
        res["conv"].add((lv, cp.in_channels, cp.out_channels, 0, 2 * Cf))
        res["conv"].add((lv, rp.in_channels, rp.out_channels + op.out_channels, Cf, 2 * Cf))
        res["head_finish"].add((nc, use_image))
        for C, ldx, off in ((nc, nc, 0), (4, 5, 0), (1, 5, 4)):
            res["to_dense"].add((C, ldx, off, use_image))
    return {k: sorted(v) for k, v in res.items()}


@lru_cache(None)
def launches(size, dataset, use_image):
    """launches_of the model of one configuration, built on the CPU"""
    import torch
    from dagr_b200.model.dagr import DAGR
    W, H = SENSOR[dataset]
    torch.manual_seed(0)
    with torch.no_grad():
        model = DAGR(config_args(size, dataset, use_image), height=H, width=W).eval()
    return launches_of(model)


@lru_cache(None)
def shipped():
    """{kind: sorted union over every configuration}; conv entries without the level: (Cin, Cout, offset, ldin)"""
    res = {k: set() for k in KINDS}
    for cfg in configs():
        for k, v in launches(*cfg).items():
            res[k] |= {t[1:] for t in v} if k == "conv" else set(v)
    return {k: sorted(v) for k, v in res.items()}


def conv_labels(size, dataset, use_image):
    """the engine's profile labels of the grid convs of one configuration"""
    return sorted({f"grid_conv_L{lv}_{ci}x{co}" for lv, ci, co, _, _ in launches(size, dataset, use_image)["conv"]})
