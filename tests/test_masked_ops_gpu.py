"""The masked row ops on their own (csrc/masked.cu): dagr_masked_lin, dagr_masked_inplace_bn and dagr_masked_isdiff through the
C-ABI on every case of tests/masked_cases.py.

Every output buffer starts as a sentinel (the base table where masked_lin adds), and then
  - the rows not selected keep their bits;
  - the selected rows equal the reference's own asy_tools kernels bit for bit (tests/golden/masked_ops_golden.npz, made by
    tests/golden/make_masked_ops_golden.py);
  - lin and bn lie within a float64 bound |got - ref64| <= c u S + 2 u |ref64| (S: the sum of the magnitudes of the terms);
  - isdiff's decisions equal the exact model (float32 |a - b| against a correctly rounded fmaf(rtol, b, atol)).
Widths cross the warp (1 .. 258 channels), K crosses the CTA tails (4 rows per CTA, 256 elements per CTA in bn), rows are
taken at the end of a 262 147-row table, and the isdiff knife edges sit at the threshold and one ulp either side."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests.masked_cases import SENTINEL, case_names, isdiff_model, make_case

pytestmark = pytest.mark.gpu

GOLD = np.load(Path(__file__).resolve().parent / "golden" / "masked_ops_golden.npz")
U = 2.0 ** -24


def _lib():
    from dagr_b200 import _lib
    return _lib, _lib.load()


def _sentinel(rows, cols):
    return torch.full((rows, cols), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def bound_ratio(out, ref, S, c):
    """max over elements of |out - ref| / (c u S + 2 u |ref|); NaN counts as infinite"""
    out, ref, S = out.double(), ref.double(), S.double()
    err = (out - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / (c * U * S + 2 * U * ref.abs()))
    r = torch.where(torch.isnan(out), torch.full_like(err, float("inf")), r)
    return float(r.max()) if r.numel() else 0.0


def run(case):
    """the kernel on the case; returns (output table or kept indices, the buffer as it was before the call)"""
    L, lib = _lib()
    m = {k: v.cuda().contiguous() if torch.is_tensor(v) else v for k, v in case.items()}
    idx, K = m["idx"], len(case["idx"])
    if case["op"] == "lin":
        R, Cout = m["base"].shape
        Cin = m["x"].shape[1]
        out = m["base"].clone() if m["add"] else _sentinel(R, Cout)
        before = out.clone()
        L.check(lib.dagr_masked_lin(L.ptr(idx), K, L.ptr(m["x"]), L.ptr(out), L.ptr(m["w"]), L.ptr(m["b"]), Cin, Cout, m["add"],
                                    L.stream_ptr()), "dagr_masked_lin")
    elif case["op"] == "bn":
        out = _sentinel(*m["x"].shape)
        before = out.clone()
        L.check(lib.dagr_masked_inplace_bn(L.ptr(idx), K, L.ptr(m["x"]), L.ptr(out), L.ptr(m["mean"]), L.ptr(m["var"]),
                                           L.ptr(m["w"]), L.ptr(m["b"]), m["x"].shape[1], m["eps"], L.stream_ptr()),
                "dagr_masked_inplace_bn")
    else:
        out = idx.clone()
        before = out.clone()
        L.check(lib.dagr_masked_isdiff(L.ptr(out), K, L.ptr(m["a"]), L.ptr(m["b"]), m["a"].shape[1], m["atol"], m["rtol"],
                                       L.stream_ptr()), "dagr_masked_isdiff")
    torch.cuda.synchronize()
    return out.cpu(), before.cpu()


def reference64(case):
    """(float64 result, S = sum of |terms|, c) of the selected rows"""
    idx = case["idx"]
    if case["op"] == "lin":
        x, w = case["x"][idx].double(), case["w"].double()
        terms = x[:, None, :] * w[None, :, :]                              # [K, Cout, Cin]
        ref, S = terms.sum(-1), terms.abs().sum(-1)
        if case["add"]:
            ref, S = ref + case["base"][idx].double(), S + case["base"][idx].double().abs()
        if case["b"] is not None:
            ref, S = ref + case["b"].double(), S + case["b"].double().abs()
        return ref, S, x.shape[1] + 2
    d = (case["x"][idx].double() - case["mean"].double()) / torch.sqrt(case["var"].double() + np.float32(case["eps"]))
    dw = d * case["w"].double()
    return dw + case["b"].double(), dw.abs() + case["b"].double().abs(), 6


@pytest.mark.parametrize("name", case_names())
def test_masked_op_against_reference_kernel_and_models(name):
    case = make_case(name)
    got, before = run(case)
    idx = case["idx"]
    gold = torch.from_numpy(GOLD[name])
    if case["op"] == "isdiff":
        assert torch.equal(got, gold), f"kept indices differ from the reference kernel at {torch.nonzero(got != gold).flatten()[:8].tolist()}"
        want = torch.from_numpy(isdiff_model(case["a"].numpy(), case["b"].numpy(), idx.numpy(), case["atol"], case["rtol"]))
        assert torch.equal(got, want)
        if "meta" in case:                                             # the knife edges decide as built
            meta = [case["meta"][r] for r in idx.tolist()]
            assert [int(k >= 0) for k in got.tolist()] == [int(off > 0) for _, off in meta]
        return
    keep = torch.ones(len(got), dtype=torch.bool)
    keep[idx] = False
    assert torch.equal(got[keep].view(torch.int32), before[keep].view(torch.int32)), "a row that is not selected changed"
    sel = got[idx]
    assert sel.shape == gold.shape
    bad = torch.nonzero(sel.view(torch.int32) != gold.view(torch.int32))
    assert len(bad) == 0, f"{len(bad)} of {sel.numel()} outputs differ from the reference kernel, first {bad[:3].tolist()}: " \
                          f"{[(float(sel[tuple(b)]), float(gold[tuple(b)])) for b in bad[:3]]}"
    if len(idx):
        ref, S, c = reference64(case)
        assert bound_ratio(sel, ref, S, c) <= 1.0
