#!/usr/bin/env python
"""Generate tests/golden/downsample_golden.npz from the REFERENCE's own down-sampler (build container only).

    DAGR_REFERENCE=/path/to/uzh-rpg/dagr python tests/golden/make_downsample_golden.py

scripts/downsample_events.py imports h5py / hdf5plugin / dsec_det at module level for its file I/O; they are stubbed so
that the numba function `downsample_events` itself runs unmodified.  Each case pushes its chunks through with the change
map carried over, as the script's main loop does (:146-153).  Keys per case c: c{c}_shape = [iw, ih, ow, oh], optional
c{c}_map0 (the change map the first chunk starts from; zeros when absent), and per chunk k c{c}_k{k}_in_{x,y,p,t},
c{c}_k{k}_out_{x,y,p,t} and c{c}_k{k}_map (the map after the chunk).

  c0..c2  three chunks each: 640x480 -> 320x240; 64x48 -> 32x24 with a hot-pixel chunk; 96x48 -> 32x24 (fx = 3, fy = 2)
  c3..c7  fx x fy = 1x1, 2x1, 3x1, 3x3, 4x2 (denominators 1, 2, 3, 9, 8), two chunks each, the map seeded near +-1
  c8      3x3, more output cells (200 x 150) than events, seeded map
  c9      4x2, one chunk of 16384 events with 7000 in one output cell (more than 3 scan tiles of 2048), seeded map

The seeds are +-1 and one float32 ulp either side, +-(1 - k/d) and one ulp either side for k = 1..3, and +-(1 - 2^-24);
the events of the seeded cases fall mostly on the seeded cells.  Every input has x < fx * ow and y < fy * oh: the numba
loop has no bounds check.  c0..c2 draw from the generator first, so appending cases leaves them unchanged.
"""
import importlib.util
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

if not os.environ.get("DAGR_REFERENCE"):
    sys.exit("set DAGR_REFERENCE to an uzh-rpg/dagr checkout")
os.environ.setdefault("NUMBA_CACHE_DIR", tempfile.mkdtemp())          # the script asks numba for an on-disk cache
for name in ("hdf5plugin", "h5py", "tqdm", "dsec_det", "dsec_det.io"):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules["h5py"].File = object                                    # only used in a type annotation
sys.modules["dsec_det.io"].extract_from_h5_by_index = None
sys.modules["dsec_det.io"].get_num_events = None
spec = importlib.util.spec_from_file_location("ref_downsample", Path(os.environ["DAGR_REFERENCE"]) / "scripts" / "downsample_events.py")
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)


def map_seeds(d):
    """float32 accumulator values at the pass decision of denominator d (all |v| < 2)."""
    one = np.float32(1)
    base = [one] + [np.float32(1 - k / d) for k in range(1, 4) if k < d] + [np.float32(1 - 2.0 ** -24)]
    v = []
    for b in base:
        v += [b, np.nextafter(b, np.float32(0)), np.nextafter(b, np.float32(2))]
    v = np.array(v, np.float32)
    return np.unique(np.concatenate([v, -v]))


rng = np.random.default_rng(7)
out = {}


def run(case, iw, ih, ow, oh, chunks, map0=None):
    """chunks: list of event dicts (x, y, p, t) at the input resolution."""
    cm = None if map0 is None else map0.copy()
    if map0 is not None:
        out[f"c{case}_map0"] = map0.copy()
    for chunk, ev in enumerate(chunks):
        fx, fy = iw // ow, ih // oh
        assert ev["x"].max() < fx * ow and ev["y"].max() < fy * oh
        res, cm = ref.downsample_events({k: v.copy() for k, v in ev.items()}, ih, iw, oh, ow, change_map=cm)
        for k, v in ev.items():
            out[f"c{case}_k{chunk}_in_{k}"] = v
        for k, v in res.items():
            out[f"c{case}_k{chunk}_out_{k}"] = v
        out[f"c{case}_k{chunk}_map"] = cm.copy()
    out[f"c{case}_shape"] = np.array([iw, ih, ow, oh])


for case, (iw, ih, ow, oh, n) in enumerate([(640, 480, 320, 240, 6000), (64, 48, 32, 24, 5000), (96, 48, 32, 24, 4000)]):
    chunks = []
    for chunk in range(3):
        ev = dict(x=rng.integers(0, iw, n).astype("uint16"), y=rng.integers(0, ih, n).astype("uint16"),
                  p=(2 * rng.integers(0, 2, n) - 1).astype("int8"), t=np.sort(rng.integers(0, 50000, n)).astype("int64") + 50000 * chunk)
        if case == 1 and chunk == 1:                                    # hot pixels: long runs on a few cells
            ev["x"][: n // 2] = 10
            ev["y"][: n // 2] = 7
            ev["p"][: n // 2 : 3] = 1
        chunks.append(ev)
    run(case, iw, ih, ow, oh, chunks)


def seeded(ow, oh, d):
    """a map with the seeds of d on its first cells (cyclically on about a third of the map), zeros elsewhere; returns
    (map, flat indices of the seeded cells)."""
    s = map_seeds(d)
    m = np.zeros(oh * ow, np.float32)
    cells = rng.permutation(oh * ow)[: max(len(s), oh * ow // 3)]
    m[cells] = s[np.arange(len(cells)) % len(s)]
    return m.reshape(oh, ow), cells


def events(n, iw, ih, fx, fy, ow, cells, t0, frac=0.8):
    """n events; a fraction `frac` of them on the output cells `cells` (anywhere inside the fx x fy input block)."""
    x, y = rng.integers(0, iw, n), rng.integers(0, ih, n)
    on = rng.random(n) < frac
    c = cells[rng.integers(0, len(cells), on.sum())]
    x[on] = (c % ow) * fx + rng.integers(0, fx, on.sum())
    y[on] = (c // ow) * fy + rng.integers(0, fy, on.sum())
    return dict(x=x.astype("uint16"), y=y.astype("uint16"), p=(2 * rng.integers(0, 2, n) - 1).astype("int8"),
                t=(t0 + np.sort(rng.integers(0, 50000, n))).astype("int64"))


case = 3
for fx, fy in ((1, 1), (2, 1), (3, 1), (3, 3), (4, 2)):
    ow, oh = 32, 24
    iw, ih = fx * ow, fy * oh
    m0, cells = seeded(ow, oh, fx * fy)
    run(case, iw, ih, ow, oh, [events(3000, iw, ih, fx, fy, ow, cells, 50000 * k) for k in range(2)], m0)
    case += 1
# more output cells than events
ow, oh, fx, fy = 200, 150, 3, 3
m0, cells = seeded(ow, oh, 9)
run(case, fx * ow, fy * oh, ow, oh, [events(1000, fx * ow, fy * oh, fx, fy, ow, cells, 0)], m0)
case += 1
# one hot cell holding 7000 of 16384 events, mixed polarities with a positive bias
ow, oh, fx, fy = 32, 24, 4, 2
m0, cells = seeded(ow, oh, 8)
ev = events(16384, fx * ow, fy * oh, fx, fy, ow, cells, 0)
hot = rng.permutation(16384)[:7000]
ev["x"][hot] = 5 * fx + rng.integers(0, fx, 7000)
ev["y"][hot] = 9 * fy + rng.integers(0, fy, 7000)
ev["p"][hot] = np.where(rng.random(7000) < 0.7, 1, -1)
run(case, fx * ow, fy * oh, ow, oh, [ev], m0)

dst = Path(__file__).parent / "downsample_golden.npz"
if dst.exists():                                                     # the committed cases must come out bit for bit the same
    old = np.load(dst)
    for k in old.files:
        if k not in out or not (old[k].dtype == out[k].dtype and np.array_equal(old[k], out[k])):
            sys.exit(f"{k} differs from the committed fixture")
np.savez_compressed(dst, **out)
print("wrote", len(out), "arrays")
