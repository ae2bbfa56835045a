"""The masked row ops without a GPU: the argument contract of dagr_masked_lin, dagr_masked_inplace_bn and dagr_masked_isdiff
(every bad input is refused with DAGR_E_ARG and a message naming the function before anything is launched), and the case
builders of tests/masked_cases.py (distinct rows, knife edges exactly where they are meant to be, exact float32 rounding)."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from tests import masked_cases as M

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first


def _lin(lib, K=3, idx=BAD, x=BAD, out=BAD, w=BAD, b=BAD, Cin=4, Cout=5):
    return lib.dagr_masked_lin(idx, K, x, out, w, b, Cin, Cout, 0, None)


def _bn(lib, K=3, idx=BAD, x=BAD, out=BAD, mean=BAD, var=BAD, w=BAD, b=BAD, C=5):
    return lib.dagr_masked_inplace_bn(idx, K, x, out, mean, var, w, b, C, 1e-5, None)


def _isdiff(lib, K=3, idx=BAD, a=BAD, b=BAD, C=5):
    return lib.dagr_masked_isdiff(idx, K, a, b, C, 1e-8, 1e-5, None)


CALLS = {"dagr_masked_lin": _lin, "dagr_masked_inplace_bn": _bn, "dagr_masked_isdiff": _isdiff}


@pytest.mark.parametrize("fn,kw,needle", [
    ("dagr_masked_lin", dict(K=-1), "K < 0"),
    ("dagr_masked_lin", dict(Cin=0), "Cin and Cout"),
    ("dagr_masked_lin", dict(Cout=0), "Cin and Cout"),
    ("dagr_masked_lin", dict(Cout=-3), "Cin and Cout"),
    ("dagr_masked_lin", dict(idx=None), "null pointer"),
    ("dagr_masked_lin", dict(x=None), "null pointer"),
    ("dagr_masked_lin", dict(out=None), "null pointer"),
    ("dagr_masked_lin", dict(w=None), "null pointer"),
    ("dagr_masked_inplace_bn", dict(K=-1), "K < 0"),
    ("dagr_masked_inplace_bn", dict(C=0), "C must be"),
    ("dagr_masked_inplace_bn", dict(idx=None), "null pointer"),
    ("dagr_masked_inplace_bn", dict(x=None), "null pointer"),
    ("dagr_masked_inplace_bn", dict(out=None), "null pointer"),
    ("dagr_masked_inplace_bn", dict(mean=None), "null pointer"),
    ("dagr_masked_inplace_bn", dict(var=None), "null pointer"),
    ("dagr_masked_inplace_bn", dict(w=None), "null pointer"),
    ("dagr_masked_inplace_bn", dict(b=None), "null pointer"),
    ("dagr_masked_isdiff", dict(K=-1), "K < 0"),
    ("dagr_masked_isdiff", dict(C=0), "C must be"),
    ("dagr_masked_isdiff", dict(idx=None), "null pointer"),
    ("dagr_masked_isdiff", dict(a=None), "null pointer"),
    ("dagr_masked_isdiff", dict(b=None), "null pointer"),
])
def test_masked_ops_reject_bad_arguments(fn, kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert CALLS[fn](lib, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert fn in msg and needle in msg, msg


@pytest.mark.parametrize("fn", sorted(CALLS))
def test_masked_ops_accept_nothing_to_do(fn):
    """K = 0 with NULL buffers is a valid empty call: nothing is launched"""
    from dagr_b200 import _lib
    lib = _lib.load()
    nulls = {"dagr_masked_lin": dict(idx=None, x=None, out=None, w=None, b=None),
             "dagr_masked_inplace_bn": dict(idx=None, x=None, out=None, mean=None, var=None, w=None, b=None),
             "dagr_masked_isdiff": dict(idx=None, a=None, b=None)}[fn]
    assert CALLS[fn](lib, K=0, **nulls) == 0


# ---- case builders --------------------------------------------------------------------------------------------------------
def test_case_names_cover_the_widths_and_ks():
    names = M.case_names()
    assert len(names) == len(set(names))
    for cin in M.CIN:
        for cout in M.COUT:
            assert f"lin_{cin}x{cout}_bias_add1" in names and f"lin_{cin}x{cout}_nobias_add0" in names
    for c in M.CS:
        assert f"bn_c{c}" in names and f"isdiff_c{c}" in names
    for k in M.KS:
        assert f"lin_k{k}_bias_add0" in names and f"bn_k{k}" in names and f"isdiff_k{k}" in names
    assert {1, 3, 31, 32, 33, 258} <= set(M.CS) and 4097 in M.KS and 0 in M.KS


@pytest.mark.parametrize("name", ["lin_33x130_bias_add1", "lin_k4097_nobias_add0", "lin_tail_bias_add1", "bn_c258", "bn_k4097",
                                  "bn_tail", "isdiff_c33", "isdiff_k5", "isdiff_tail", "isdiff_edges_c33", "isdiff_specials"])
def test_cases_select_distinct_rows_inside_the_table(name):
    c = M.make_case(name)
    rows = (c["x"] if c["op"] != "isdiff" else c["a"]).shape[0]
    idx = c["idx"].tolist()
    assert len(set(idx)) == len(idx) and all(0 <= r < rows for r in idx)
    if "tail" in name:
        assert rows == M.TAIL_ROWS and rows - 1 in idx
    assert M.make_case(name)["idx"].tolist() == idx                     # seeded: the same case every time


@pytest.mark.parametrize("C", M.EDGE_C)
def test_isdiff_knife_edges_are_exact(C):
    c = M.make_case(f"isdiff_edges_c{C}")
    a, b = c["a"].numpy(), c["b"].numpy()
    seen = set()
    for r, (pos, off) in enumerate(c["meta"]):
        for ch in range(C):
            T = Fraction(float(M.fma32(c["rtol"], b[r, ch], c["atol"])))
            assert T == M.round_f32(Fraction(float(np.float32(c["rtol"]))) * Fraction(float(b[r, ch])) +
                                    Fraction(float(np.float32(c["atol"]))))
            d = abs(Fraction(float(a[r, ch])) - Fraction(float(b[r, ch])))
            assert Fraction(float(np.abs(a[r, ch] - b[r, ch]))) == d        # the float32 subtraction is exact
            want = off if ch == pos else 0
            assert (d > T) - (d < T) == want
            if want:
                assert abs(d - T) == Fraction(float(np.spacing(np.float32(max(d, T))) if want < 0 else
                                                    np.spacing(np.float32(T))))
        seen.add((pos, off, bool(b[r, pos] < 0), bool(a[r, pos] < b[r, pos])))
    assert {p for p, _, _, _ in seen} == {0, 31, 32, C - 1}
    assert len(seen) == len({0, 31, 32, C - 1}) * 3 * 2 * 2              # every position x offset x sign of b x sign of D
    want = [r if c["meta"][r][1] > 0 else -1 for r in c["idx"].tolist()]
    assert M.isdiff_model(a, b, c["idx"].numpy(), c["atol"], c["rtol"]).tolist() == want


def test_isdiff_model_signed_threshold_and_non_finite_values():
    c = M.make_case("isdiff_specials")
    a, b = c["a"].numpy(), c["b"].numpy()
    got = M.isdiff_model(a, b, np.arange(len(a)), c["atol"], c["rtol"])
    for r in range(len(a)):
        bad = [ch for ch in range(a.shape[1]) if not (a[r, ch] == b[r, ch])]
        if not bad:
            assert got[r] == -1
            continue
        va, vb = a[r, bad[0]], b[r, bad[0]]
        changed = not np.isnan(va) and not np.isnan(vb) and not (np.isinf(va) and va == vb) and vb != np.inf
        assert (got[r] >= 0) == changed, (va, vb)
    q3 = M.make_case("isdiff_c33")                                        # b = a = -2: 0 > atol - 2 rtol, a change
    r = int(q3["idx"][1])
    assert q3["a"][r, 0] == q3["b"][r, 0] == -2.0
    assert M.isdiff_model(q3["a"].numpy(), q3["b"].numpy(), [r], q3["atol"], q3["rtol"])[0] == r


def test_round_f32_rounds_once():
    one = Fraction(1)
    h = Fraction(1, 2 ** 24)                                              # half an ulp of 1.0f
    assert M.round_f32(one + h) == np.float32(1.0)                        # tie: to even
    assert M.round_f32(one + 3 * h) == np.float32(1 + 2.0 ** -22)         # tie: to even, upwards
    # just above the tie: float64 would round to the tie first and then to 1.0f
    above = one + h + Fraction(1, 2 ** 80)
    assert np.float32(float(above)) == np.float32(1.0) and M.round_f32(above) == np.float32(1 + 2.0 ** -23)
    rng = np.random.default_rng(0)
    x, y = (rng.standard_normal(2000).astype(np.float32) for _ in range(2))
    z = rng.standard_normal(2000).astype(np.float32)
    for xi, yi, zi in zip(x, y, z):                                      # exact in float64 at these magnitudes: one rounding
        p = np.float64(xi) * np.float64(yi)
        if abs(p) > 2.0 ** -4 and abs(zi) > 2.0 ** -4 and max(abs(p), abs(zi)) / min(abs(p), abs(zi)) < 16:
            assert M.fma32(xi, yi, zi) == np.float32(p + np.float64(zi))
