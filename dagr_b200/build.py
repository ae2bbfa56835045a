"""In-tree build of libdagr_b200.so (hand-written sm_90a kernels for the H100 behind a C-ABI, no torch headers).

    python -m dagr_b200.build          # nvcc -gencode arch=compute_90a,code=sm_90a -> dagr_b200/libdagr_b200.so
"""
import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libdagr_b200.so"
SOURCES = ["capi.cu", "graph.cu", "build_l1.cu", "conv_l1.cu", "image_l1.cu", "coarse.cu", "masked.cu", "ingest.cu", "evaluate.cu", "labels.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17"] + GENCODE + ["-lineinfo",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


HASHFILE = PKG / "libdagr_b200.srchash"


def _source_hash() -> str:
    import hashlib
    h = hashlib.sha256()
    deps = [CSRC / s for s in SOURCES] + sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "dagr_b200.h"]
    for d in deps:
        h.update(d.name.encode())
        h.update(d.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def needs_build() -> bool:
    """the library is stale when the sources' content hash differs from the one recorded at build time (mtimes do not
    survive a copy of the tree to another box)."""
    if not LIB.exists() or not HASHFILE.exists():
        return True
    return HASHFILE.read_text().strip() != _source_hash()


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    objs = []
    nvcc = _nvcc()
    bdir = PKG / "build"
    bdir.mkdir(exist_ok=True)
    procs = []
    for s in SOURCES:
        o = bdir / (s.replace(".cu", ".o"))
        cmd = [nvcc, "-c", str(CSRC / s), "-o", str(o)] + NVCC_FLAGS
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(str(o))
    log = []
    for s, p in procs:
        out, _ = p.communicate()
        log.append(f"== {s}\n{out}")
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{out}")
    (bdir / "ptxas.log").write_text("\n".join(log))
    cmd = [nvcc, "-shared", "-o", str(LIB)] + objs + GENCODE + ["-lcudart"]
    subprocess.check_call(cmd)
    HASHFILE.write_text(_source_hash() + "\n")
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="-f" in sys.argv, verbose="-v" in sys.argv))
