#!/usr/bin/env python
"""Generate tests/golden/masked_ops_golden.npz from the REFERENCE's own asy_tools kernels (needs a GPU and oracle/_ref, see
oracle/build_ref.py): masked_lin / masked_lin_no_bias / masked_inplace_BN / masked_isdiff on every case of
tests/masked_cases.py.  Stored per case: the selected rows of the output (lin, bn), or the index array masked_isdiff leaves
in place (the row index or -1 per selected row).  K = 0 is not launched (the reference would launch an empty grid); its
entry is empty.

    python tests/golden/make_masked_ops_golden.py [OUT.npz]
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "_ref" / "asy_tools"))
import asy_tools                                                     # noqa: E402

from tests.masked_cases import SENTINEL, case_names, make_case       # noqa: E402


def sentinel(rows, cols, dev):
    return torch.full((rows, cols), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def run(case, dev="cuda"):
    m = {k: v.to(dev).contiguous() if torch.is_tensor(v) else v for k, v in case.items()}
    idx = m["idx"]
    if case["op"] == "lin":
        R, Cout = m["base"].shape
        o = m["base"].clone() if m["add"] else sentinel(R, Cout, dev)
        if len(idx):
            if m["b"] is None:
                asy_tools.masked_lin_no_bias(idx, m["x"], o, m["w"], bool(m["add"]))
            else:
                asy_tools.masked_lin(idx, m["x"], o, m["w"], m["b"], bool(m["add"]))
        return o[idx].cpu().numpy()
    if case["op"] == "bn":
        o = sentinel(*m["x"].shape, dev)
        if len(idx):
            asy_tools.masked_inplace_BN(idx, m["x"], o, m["mean"], m["var"], m["w"], m["b"], m["eps"])
        return o[idx].cpu().numpy()
    kept = idx.clone()
    if len(idx):
        asy_tools.masked_isdiff(kept, m["a"], m["b"], m["atol"], m["rtol"])
    return kept.cpu().numpy()


if __name__ == "__main__":
    out = {name: run(make_case(name)) for name in case_names()}
    torch.cuda.synchronize()
    out["device"] = np.array(torch.cuda.get_device_name())
    dst = Path(sys.argv[1]) if len(sys.argv) > 1 else Path(__file__).parent / "masked_ops_golden.npz"
    dst.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(dst, **out)
    print("wrote", dst, len(out), "entries,", sum(v.nbytes for v in out.values()), "bytes")
