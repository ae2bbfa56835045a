"""k_grid_conv_tiled, the large-grid kernel of dagr_grid_conv, at every tile size it can choose.

The kernel picks M (voxels per CTA) from the cell count, and its bits must not depend on M.  For each M, a batch sized to
land on that M with a partial last tile, empty samples and empty cells runs through the large-grid kernel; the rows of
the samples in two windows of it (one ending at the partial last tile) must equal, bit for bit, the same samples run as
a batch small enough for k_grid_conv_sk<4>.  Shapes: 18x64, 64x64, 66x64 (Cin not a multiple of 4 or 8), 18x128 (two
column tiles), and the column blocks 32x100 and 64x5 (ldin = 2 Cin, Cout not a multiple of 4 and one partial tile).
"""
import numpy as np
import pytest
import torch

from tests.test_grid_kernels_cpu import make_grid
from tests.test_grid_kernels_gpu import conv_params, instance, n_sm, real_den, run_grid_conv

pytestmark = pytest.mark.gpu

NX, NY = 13, 7
PER = NX * NY
TILES = (16, 32, 48, 64)
SHAPES = [(18, 64, False), (64, 64, False), (66, 64, False), (18, 128, False), (32, 100, True), (64, 5, True)]
SMALL = 12                                            # samples in a reference batch (1092 cells: k_grid_conv_sk<4>)


def tile(cells, nsm):
    """the M that k_grid_conv_tiled runs at (coarse.cu: grid_conv_tile): fewest voxels on the busiest SM, larger M on a tie"""
    best, best_m = None, None
    for m in (64, 48, 32, 16):
        ctas = -(-cells // m)
        load = -(-ctas // nsm) * m
        if best is None or load < best:
            best, best_m = load, m
    return best_m


def batch_for_tile(m, nsm):
    """the least number of samples whose grid takes the large-grid kernel at tile M with a partial last tile"""
    for B in range(1, 4096):
        cells = B * PER
        if cells >= 32 * nsm and tile(cells, nsm) == m and cells % m:
            return B
    raise AssertionError(f"no batch of {PER}-cell samples reaches M = {m} on {nsm} SMs")


def sample(i, Cin, Cout, ldin, off, empty):
    """sample i: its grid (40 % empty cells, or all of them), input rows (a column block when ldin), skip rows"""
    rng = np.random.default_rng([i, Cin, Cout])
    den = real_den()
    cnt, pxy, mask = make_grid(rng, NX, NY, 1, [] if empty else [0], px_max=int(den[0]) // 2, py_max=int(den[1]) // 2)
    x = np.full((PER, ldin or Cin), np.nan, np.float32)
    x[:, off:off + Cin] = rng.standard_normal((PER, Cin))
    return dict(cnt=cnt, pxy=pxy, mask=mask, x=x, skip=rng.standard_normal((PER, Cout)).astype(np.float32))


def run(samples, Cin, Cout, ldin, off, p):
    B = len(samples)
    g = dict(nx=NX, ny=NY, B=B, den_x=real_den()[0], den_y=real_den()[1],
             **{k: np.concatenate([s[k] for s in samples]) for k in ("cnt", "pxy", "mask")})
    q = dict(p, skip=np.concatenate([s["skip"] for s in samples]))
    out, seen = run_grid_conv(g, np.concatenate([s["x"] for s in samples]), off, ldin, Cin, Cout, q)
    return out, seen


@pytest.mark.parametrize("m", TILES)
@pytest.mark.parametrize("Cin,Cout,block", SHAPES, ids=[f"{ci}x{co}{'-block' if b else ''}" for ci, co, b in SHAPES])
def test_tile_size_does_not_change_a_sample(Cin, Cout, block, m):
    nsm = n_sm()
    B = batch_for_tile(m, nsm)
    assert instance(Cin, Cout, B * PER, nsm) == "sk16" and instance(Cin, Cout, SMALL * PER, nsm) == "sk4"
    off, ldin = (Cin, 2 * Cin) if block else (0, 0)
    samples = [sample(i, Cin, Cout, ldin, off, empty=i % 5 == 3 and i < B - 1) for i in range(B)]
    p, _ = conv_params(np.random.default_rng([Cin, Cout]), "realistic", 0, Cin, Cout, ("bias", "scale", "skip"))
    big, seen = run(samples, Cin, Cout, ldin, off, p)
    assert seen == {"sk16"}
    assert not big.isnan().any() and (big[(B - 1) * PER:] != 0).any()
    for lo in (B // 2 - SMALL // 2, B - SMALL):                     # a window in the middle, one ending at the last tile
        small, seen_s = run(samples[lo:lo + SMALL], Cin, Cout, ldin, off, p)
        assert seen_s == {"sk4"}
        want = big[lo * PER:(lo + SMALL) * PER]
        assert torch.equal(small, want), (f"{Cin}x{Cout} at M = {m} (B = {B}): {int((small != want).sum())} elements of "
                                          f"samples {lo}.. differ from the same samples at B = {SMALL}")
