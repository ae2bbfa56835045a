"""writes profiles/sass_{l1_build,conv_b2}.txt: SASS of the two hot kernels (cuobjdump of the in-tree .so) preceded by an
instruction histogram (the mnemonics that matter for the design claims: FFMA, uniform constant weight loads, LDS,
1-D TMA bulk copies UBLKCP + mbarrier SYNCS, the 3xTF32 HMMA of conv_b2's phase 2).  conv_b2 = the PLAIN tensor-core instance
the headline runs."""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
so = ROOT / "dagr_b200" / "libdagr_b200.so"
txt = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True).stdout
funcs = re.split(r"(?=\t\tFunction : )", txt)
want = {"l1_build": "_Z10k_l1_buildILi1536ELi5E", "conv_b2": "_Z12k_l1_conv_b2I17dagr_l1b_params_tLi2ELb0ELb0ELb1ELb1E"}
for tag, prefix in want.items():
    body = next(f for f in funcs if f.lstrip().startswith("Function : " + prefix))
    hist = collections.Counter()
    for line in body.splitlines():
        m = re.search(r"/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m:
            op = m.group(1)
            keep_suffix = op.startswith(("LDCU", "LDS", "UBLKCP", "SYNCS", "STS", "LDG", "STG"))
            hist[op if keep_suffix else op.split(".")[0]] += 1
    total = sum(hist.values())
    out = [f"# SASS of {prefix}... from dagr_b200/libdagr_b200.so (sm_90a), {total} instructions", "# instruction histogram (top 40):"]
    out += [f"#   {n:6d}  {k}" for k, n in hist.most_common(40)]
    tensor = [k for k in hist if k.startswith(("HGMMA", "HMMA", "IMMA", "QGMMA", "UTMALDG"))]
    out.append(f"# tensor-core / tensor-map instructions: {tensor or 'none'}")
    out.append("")
    # listing without the encoding columns: "/*addr*/ INSTR ;"
    lines = []
    for line in body.splitlines():
        m = re.match(r"\s+(/\*[0-9a-f]{4,6}\*/\s+.*?;)\s*/\*", line)
        if m:
            lines.append("    " + re.sub(r"\s{2,}", "  ", m.group(1)))
        elif "Function :" in line or ".headerflags" in line:
            lines.append(line.strip())
    (ROOT / "profiles" / f"sass_{tag}.txt").write_text("\n".join(out + lines) + "\n")
    print(tag, total, hist.most_common(12))
