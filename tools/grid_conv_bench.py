#!/usr/bin/env python
"""dagr_grid_conv on its own: CUDA-event time per launch of the pooled-grid SplineConv at config 2's large-grid shapes,
two builds of the library alternated in one process.

    python tools/grid_conv_bench.py OUT --lib-a dagr_b200/build/variants/parent.so --lib-b dagr_b200/libdagr_b200.so

One seeded forward of config 2 (dagr-s, 640x480, 300000 uniform events per sample, batch 8; the same model and first
batch as bench.py's headline) records the arguments of every dagr_grid_conv launch on the level-1 and level-2 grids
(pooled grid, input rows, skip rows, weights).  Beside those, 18 -> 128 and the column blocks 32 -> 100 and 64 -> 5
(ldin = 2 Cin) run on the level-1 grid with seeded random rows and weights.  Every case runs --launches launches per
library per round after 10 warm-up launches, libraries alternated (order swapped every round), --rounds rounds; the
median, min and max of the per-round ms per launch are reported, with executed GFLOP/s = 2 * cells * 26 * Cin * Cout /
time (the slot form every kernel executes) and whether the two libraries' outputs are the same bits.  The card's name and
power limit are read in the same run.  Writes OUT/h100_grid_conv.json.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

W, H = 640, 480


def load(path):
    from dagr_b200 import _lib
    lib = C.CDLL(str(path))
    for name in ("dagr_grid_conv", "dagr_grid_conv_last_instance"):
        res, args = _lib._SIGS[name]
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def capture_config2():
    """{label: launch arguments} of the level-1 and level-2 grid convs of one config-2 forward (first launch per label)"""
    from dagr_b200.data import format_data, synth_batch
    from dagr_b200.model.dagr import DAGR
    from dagr_b200.utils.args import default_args
    from tests.helpers import randomize_bn
    torch.manual_seed(0)
    model = randomize_bn(DAGR(default_args("s", batch_size=8), height=H, width=W).eval()).cuda()
    data = format_data(synth_batch(8, 300_000, W, H, seed=42 + 1000 * 2, kind="uniform").cuda())
    eng = model.engine
    eng.overlap = False
    cases, orig = {}, eng._grid_conv

    def hook(geom, lv, gs, xin, pack, skip, out, st, ldin=0):
        label = f"grid_conv_L{lv + 1}_{pack.cin}x{pack.cout}"
        if lv <= 1 and label not in cases:
            torch.cuda.synchronize()
            level = geom.levels[lv]
            cases[label] = dict(grid=level.grid, den=(level.den_x, level.den_y), cnt=gs.cnt.clone(), pxy=gs.pxy.clone(),
                                mask=gs.mask.clone(), x=xin.clone(), ldin=int(ldin), cin=pack.cin, cout=pack.cout,
                                w=pack.weight, root=pack.rootT, bias=pack.bias, scale=pack.scale, shift=pack.shift,
                                skip=None if skip is None else skip.clone(), relu=1 if pack.relu else 0, off=0)
        return orig(geom, lv, gs, xin, pack, skip, out, st, ldin)

    eng._grid_conv = hook
    with torch.no_grad():
        model.forward_decoded(data)
    torch.cuda.synchronize()
    eng._grid_conv = orig
    return cases


def synthetic(base, cin, cout, block, seed):
    """cin -> cout on the grid of `base` with seeded random rows and weights; block: columns [cin, 2 cin) of [cells, 2 cin]"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    cells = base["cnt"].numel()
    ld = 2 * cin if block else cin
    rnd = lambda *s: torch.randn(*s, generator=g).cuda()                    # noqa: E731
    return dict(base, x=rnd(cells, ld), ldin=ld if block else 0, off=cin if block else 0, cin=cin, cout=cout,
                w=rnd(25, cin, cout) / (2 * cin ** 0.5), root=rnd(cin, cout) / cin ** 0.5, bias=rnd(cout), scale=rnd(cout),
                shift=rnd(cout), skip=None, relu=1)


def launch(lib, c, out):
    x = c["x"][:, c["off"]:] if c["off"] else c["x"]
    rc = lib.dagr_grid_conv(c["grid"], c["cnt"], c["pxy"], c["mask"], x, c["ldin"], c["cin"], c["cout"], c["w"], c["root"],
                            c["bias"], c["scale"], c["shift"], c["skip"], c["relu"], c["den"][0], c["den"][1], out,
                            torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc


def time_launches(lib, c, out, n):
    for _ in range(10):
        launch(lib, c, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        launch(lib, c, out)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", help="directory that receives h100_grid_conv.json")
    ap.add_argument("--lib-a", required=True, help="library A (e.g. the parent commit's build)")
    ap.add_argument("--lib-b", required=True, help="library B (e.g. this tree's build)")
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "grid_conv_bench times device kernels: it needs a CUDA device"
    assert a.launches >= 200
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    libs = {"a": load(a.lib_a), "b": load(a.lib_b)}
    cases = capture_config2()
    base = cases["grid_conv_L1_64x64"]
    cases["L1_grid_18x128"] = synthetic(base, 18, 128, False, 1)
    cases["L1_grid_32x100_block"] = synthetic(base, 32, 100, True, 2)
    cases["L1_grid_64x5_block"] = synthetic(base, 64, 5, True, 3)
    res = {"gpu": gpu, "lib_a": str(a.lib_a), "lib_b": str(a.lib_b), "launches_per_round": a.launches, "rounds": a.rounds,
           "fp32_flop": "executed slot form 2 * cells * 26 * Cin * Cout", "cases": {}}
    for name, c in cases.items():
        cells = c["cnt"].numel()
        outs = {k: torch.full((cells, c["cout"]), float("nan"), device="cuda") for k in libs}
        ms = {k: [] for k in libs}
        inst = {}
        for r in range(a.rounds):
            for k in (("a", "b") if r % 2 == 0 else ("b", "a")):
                ms[k].append(time_launches(libs[k], c, outs[k], a.launches))
                inst[k] = libs[k].dagr_grid_conv_last_instance()
        flop = 2.0 * cells * 26 * c["cin"] * c["cout"]
        row = {"cells": cells, "cin": c["cin"], "cout": c["cout"], "ldin": c["ldin"], "instance": inst,
               "same_bits": bool(torch.equal(outs["a"], outs["b"]))}
        for k in libs:
            s = sorted(ms[k])
            row[k] = {"ms_median": s[len(s) // 2], "ms_min": s[0], "ms_max": s[-1],
                      "tflops_executed": flop / (s[len(s) // 2] * 1e-3) / 1e12}
        row["speedup"] = row["a"]["ms_median"] / row["b"]["ms_median"]
        res["cases"][name] = row
        print(name, json.dumps(row), flush=True)
    heads = [k for k in res["cases"] if k.startswith("grid_conv_L")]
    res["headline_sum_ms"] = {k: sum(res["cases"][h][k]["ms_median"] for h in heads) for k in libs}
    print("sum of", heads, res["headline_sum_ms"], flush=True)
    Path(a.out).mkdir(parents=True, exist_ok=True)
    (Path(a.out) / "h100_grid_conv.json").write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
