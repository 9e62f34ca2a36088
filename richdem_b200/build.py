"""Build recipe for librichdem_b200.so (nvcc, sm_90a only, in-tree)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "librichdem_b200.so")
SOURCES = ["capi.cu", "comm.cu", "fill.cu", "flats.cu", "flowdirs.cu", "accum.cu", "terrain.cu", "attributes.cu", "depressions.cu",
           "f64.cu", "f64_band.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O2,-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]
# compile-time tuning knobs of the fill sweep (tile shape, CTA size), e.g. RDB_DEFS="-DRDB_TY=32"
NVCC_FLAGS += os.environ.get("RDB_DEFS", "").split()


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [
        os.path.join(HERE, "..", "include", "richdem_b200.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    procs = []
    objs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed for {src} ---\n{out}\n")
        elif verbose and out:
            sys.stderr.write(f"--- {src} ---\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    link = [nvcc, "-shared", *GENCODE, "-o", LIB, *objs,
            "-Xcompiler", "-fPIC", "-cudart", "shared", "-ldl"]
    subprocess.check_call(link)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
