"""Seeded inputs of the masked row ops (dagr_masked_lin, dagr_masked_inplace_bn, dagr_masked_isdiff), shared by
tests/golden/make_masked_ops_golden.py, which runs the reference's own asy_tools kernels on them, and by the tests, which
compare the kernels with that fixture and with float64 / exact models.

A case is a dict: op ('lin', 'bn' or 'isdiff'), the CPU tensors the op reads, and its scalars.  Row indices are distinct
(the ops' precondition).  The isdiff knife edges are built with exact rational arithmetic: |a - b| equals
fma(rtol, b, atol) rounded to float32, or one ulp either side, in one deciding channel."""
from fractions import Fraction

import numpy as np
import torch

CIN = (1, 3, 31, 32, 33, 258)
COUT = (1, 16, 31, 32, 33, 130, 258)
CS = tuple(sorted(set(CIN) | set(COUT)))              # bn and isdiff widths
KS = (0, 1, 3, 4, 5, 4097)                           # four rows per CTA in lin / isdiff, 256 elements per CTA in bn
TAIL_ROWS = 262_147                                  # "large table": rows picked at its end
EPS = 1e-5
ATOL, RTOL = 1e-8, 1e-5
EDGE_ATOL, EDGE_RTOL = 1e-2, 1e-5                    # knife edges: |b| < 2^-8 keeps a = b +- D exact (see isdiff_edges)
EDGE_C = (33, 40)
SENTINEL = 0x7FC0BAD5                                 # a quiet-NaN bit pattern no kernel computes


def _gen(name):
    return torch.Generator().manual_seed(int.from_bytes(name.encode(), "little") % (2 ** 63))


def _rows(g, R, K, tail=False):
    if tail:                                          # the last rows of the table and row 0, shuffled
        pick = torch.tensor([R - 1, R - 2, 0, R - 3, R - 5, R - 4, R - 33])[:K]
        return pick[torch.randperm(len(pick), generator=g)]
    return torch.randperm(R, generator=g)[:K]


def lin_case(name, Cin, Cout, K, bias, add, tail=False):
    g = _gen(name)
    R = TAIL_ROWS if tail else 2 * K + 7
    return dict(op="lin", name=name, idx=_rows(g, R, K, tail), x=torch.randn(R, Cin, generator=g),
                w=torch.randn(Cout, Cin, generator=g), b=torch.randn(Cout, generator=g) if bias else None,
                base=torch.randn(R, Cout, generator=g), add=int(add))


def bn_case(name, C, K, tail=False):
    g = _gen(name)
    R = TAIL_ROWS if tail else 2 * K + 7
    x = torch.randn(R, C, generator=g)
    mean, var = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.25
    w = torch.randn(C, generator=g)
    b = torch.randn(C, generator=g)
    # half the channels: bias close to -d * w on row idx[0], so d * w + b cancels there (where an unfused multiply-add
    # shows most)
    idx = _rows(g, R, K, tail)
    if K > 0:
        r = int(idx[0])
        d = (x[r].double() - mean.double()) / torch.sqrt(var.double() + EPS)
        near = -(d * w.double()) * (1 + 1e-3 * torch.randn(C, generator=g, dtype=torch.float64))
        b = torch.where(torch.arange(C) % 2 == 0, near.float(), b)
    return dict(op="bn", name=name, idx=idx, x=x, mean=mean, var=var, w=w, b=b, eps=EPS)


def isdiff_case(name, C, K, tail=False):
    """each row: channels equal or differing by less than the threshold, and on about half the rows one channel changed by
    far more; row 1 carries the signed rtol * b quirk (b = -2 in channel 0: the threshold is negative)"""
    g = _gen(name)
    R = TAIL_ROWS if tail else 2 * K + 7
    a = torch.rand(R, C, generator=g) + 0.5
    b = a.clone()
    idx = _rows(g, R, K, tail)
    for i, r in enumerate(idx.tolist()):
        c = int(torch.randint(0, C, (1,), generator=g))
        kind = i % 4
        if kind == 1:                                 # a small change everywhere, under atol + rtol * b
            b[r] = a[r] + 1e-6 * a[r]
            b[r] = torch.where(torch.rand(C, generator=g) < 0.5, b[r], a[r])
        elif kind in (2, 3):                          # one channel far off
            b[r, c] += 0.25
    if K > 1:
        r = int(idx[1])
        a[r, 0] = b[r, 0] = -2.0                      # |a - b| = 0 > atol + rtol * (-2) < 0: changed (quirk Q3)
    return dict(op="isdiff", name=name, idx=idx, a=a, b=b, atol=ATOL, rtol=RTOL)


# ---- exact float32 arithmetic for the isdiff models ---------------------------------------------------------------------
def round_f32(q: Fraction) -> np.float32:
    """q rounded to nearest float32, ties to even (exact: no double rounding through float64)"""
    c = np.float32(float(q))
    best = None
    for v in (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))):
        if not np.isfinite(v):
            continue
        dist = abs(Fraction(float(v)) - q)
        even = (int(np.array(v).view(np.uint32)) & 1) == 0
        if best is None or dist < best[0] or (dist == best[0] and even):
            best = (dist, v)
    return best[1]


def fma32(x, y, z) -> np.float32:
    """fmaf(x, y, z) of float32 scalars, correctly rounded; IEEE results for non-finite operands"""
    x, y, z = np.float32(x), np.float32(y), np.float32(z)
    if not (np.isfinite(x) and np.isfinite(y) and np.isfinite(z)):
        return np.float32(np.float64(x) * np.float64(y) + np.float64(z))
    return round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))


def isdiff_model(a, b, idx, atol, rtol):
    """exact model of the isdiff decision: row idx[i] stays iff some channel has fl(|a - b|) > fmaf(rtol, b, atol)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    out = []
    for r in np.asarray(idx).tolist():
        with np.errstate(invalid="ignore"):
            d = np.abs(a[r] - b[r])
            t64 = np.float64(np.float32(rtol)) * b[r].astype(np.float64) + np.float64(np.float32(atol))
            clear = np.isfinite(t64) & (np.abs(d - t64) > 2.0 ** -20 * np.abs(t64))   # far from the threshold: no rounding
        keep = any(bool(d[c] > t64[c]) if clear[c] else bool(d[c] > fma32(rtol, b[r, c], atol)) for c in range(a.shape[1]))
        out.append(r if keep else -1)
    return np.array(out, dtype=np.int64)


def _step(v, n):
    for _ in range(abs(n)):
        v = np.nextafter(v, np.float32(np.inf if n > 0 else -np.inf))
    return v


def isdiff_edges(name, C):
    """knife edges: on every row each channel has |a - b| exactly at its own threshold T = fmaf(rtol, b, atol) (not a
    change: the test is strict), except the deciding channel, where |a - b| is T - 1 ulp, T or T + 1 ulp.  The deciding
    channel is 0, 31, 32 or C - 1, b is positive or negative (the threshold depends on b's sign) and a = b + D or b - D.
    b = k * 2^-30 with |b| < 2^-8 and D in [2^-7, 2^-6): a = b +- D is a float32 on the 2^-30 grid, so fl(a - b) = +-D."""
    g = _gen(name)
    rows_a, rows_b, meta = [], [], []
    grid = Fraction(1, 2 ** 30)

    def channel(sign_b, sign_d, off):
        k = int(torch.randint(2 ** 10, 2 ** 22, (1,), generator=g)) * sign_b
        bv = np.float32(float(k * grid))
        T = fma32(EDGE_RTOL, bv, EDGE_ATOL)
        D = _step(T, off)
        av = np.float32(float(Fraction(float(bv)) + sign_d * Fraction(float(D))))
        assert Fraction(float(av)) - Fraction(float(bv)) == sign_d * Fraction(float(D))
        return av, bv

    for pos in sorted({0, 31, 32, C - 1}):
        for off in (-1, 0, 1):
            for sign_b in (1, -1):
                for sign_d in (1, -1):
                    ra, rb = np.empty(C, np.float32), np.empty(C, np.float32)
                    for c in range(C):
                        if c == pos:
                            ra[c], rb[c] = channel(sign_b, sign_d, off)
                        else:
                            ra[c], rb[c] = channel(1 if c % 2 else -1, 1 if c % 3 else -1, 0)
                    rows_a.append(ra)
                    rows_b.append(rb)
                    meta.append((pos, off))
    R = len(rows_a)
    idx = torch.randperm(R, generator=g)
    return dict(op="isdiff", name=name, idx=idx, a=torch.from_numpy(np.stack(rows_a)), b=torch.from_numpy(np.stack(rows_b)),
                atol=EDGE_ATOL, rtol=EDGE_RTOL, meta=meta)


def isdiff_specials(name, C=40):
    """one non-finite value per row, at channel 0, 31, 32 or C - 1, every other channel equal: NaN in a or b (never a
    change), +-inf in a against a finite b (a change), b = +inf (threshold +inf: not a change), b = -inf (threshold -inf:
    a change), both +inf (inf - inf = NaN: not a change); and rows that are equal everywhere"""
    g = _gen(name)
    nan, inf = float("nan"), float("inf")
    kinds = [(nan, None), (None, nan), (nan, nan), (inf, None), (-inf, None), (None, inf), (None, -inf), (inf, inf), (-inf, -inf),
             (None, None)]
    rows_a, rows_b = [], []
    for pos in (0, 31, 32, C - 1):
        for va, vb in kinds:
            ra = (torch.rand(C, generator=g) + 0.5).numpy()
            rb = ra.copy()
            if va is not None:
                ra[pos] = va
            if vb is not None:
                rb[pos] = vb
            rows_a.append(ra)
            rows_b.append(rb)
    idx = torch.randperm(len(rows_a), generator=g)
    return dict(op="isdiff", name=name, idx=idx, a=torch.from_numpy(np.stack(rows_a)), b=torch.from_numpy(np.stack(rows_b)),
                atol=ATOL, rtol=RTOL)


def case_names():
    names = []
    for cin in CIN:
        for cout in COUT:
            names += [f"lin_{cin}x{cout}_{t}_add{a}" for t in ("bias", "nobias") for a in (0, 1)]
    names += [f"lin_k{k}_{t}_add{a}" for k in KS for t in ("bias", "nobias") for a in (0, 1)]
    names += [f"lin_tail_{t}_add{a}" for t in ("bias", "nobias") for a in (0, 1)]
    names += [f"bn_c{c}" for c in CS] + [f"bn_k{k}" for k in KS] + ["bn_tail"]
    names += [f"isdiff_c{c}" for c in CS] + [f"isdiff_k{k}" for k in KS] + ["isdiff_tail"]
    names += [f"isdiff_edges_c{c}" for c in EDGE_C] + ["isdiff_specials"]
    return names


def make_case(name):
    p = name.split("_")
    if p[0] == "lin":
        bias, add = p[-2] == "bias", int(p[-1][3:])
        if p[1] == "tail":
            return lin_case(name, 33, 33, 7, bias, add, tail=True)
        if p[1].startswith("k"):
            return lin_case(name, 5, 3, int(p[1][1:]), bias, add)
        cin, cout = (int(v) for v in p[1].split("x"))
        return lin_case(name, cin, cout, 5, bias, add)
    if p[0] == "bn":
        if p[1] == "tail":
            return bn_case(name, 33, 7, tail=True)
        return bn_case(name, int(p[1][1:]), 5) if p[1].startswith("c") else bn_case(name, 7, int(p[1][1:]))
    if p[1] == "tail":
        return isdiff_case(name, 33, 7, tail=True)
    if p[1] == "edges":
        return isdiff_edges(name, int(p[2][1:]))
    if p[1] == "specials":
        return isdiff_specials(name)
    return isdiff_case(name, int(p[1][1:]), 9) if p[1].startswith("c") else isdiff_case(name, 33, int(p[1][1:]))
