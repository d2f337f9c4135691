"""Build the in-tree native libraries (sm_90a only: H100).

  libcfb200.so        CUDA kernels + C ABI (include/cfb200.h) + host driver
  centrifuge-class    drop-in CLI (same name as the reference binary), links libcfb200.so

The built artefacts stay inside centrifuge_b200/ (git-ignored), where capi.py loads them.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcfb200.so")
CLI = os.path.join(HERE, "centrifuge-class")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function,-Wno-deprecated-declarations,-ffp-contract=off", "--expt-relaxed-constexpr",
    "-Wno-deprecated-gpu-targets", "-diag-suppress", "1444",
]

LIB_SOURCES = ["cfb200.cu", "cf_build.cu", "cf_em.cu", "cf_gunzip.cu", "cf_bunzip2.cu", "cf_index.cpp", "cf_host.cpp"]
CLI_SOURCES = ["cf_cli.cpp"]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    deps = list(sources) + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    deps.append(os.path.join(HERE, "..", "include", "cfb200.h"))
    deps.append(os.path.abspath(__file__))
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(verbose=False, force=False, ptxas_v=False):
    nvcc = _nvcc()
    srcs = [os.path.join(CSRC, s) for s in LIB_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    if force or _newer(LIB, srcs):
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if ptxas_v else []) + ["-shared", "-o", LIB] + srcs + ["-lcudart", "-lpthread"]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed building libcfb200.so")
    cli_srcs = [os.path.join(CSRC, s) for s in CLI_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    if cli_srcs and (force or _newer(CLI, cli_srcs + [LIB])):
        cmd = [nvcc, "-O2", "-std=c++17", "-o", CLI] + cli_srcs + ["-L" + HERE, "-lcfb200", "-Xlinker", "-rpath=$ORIGIN", "-lcudart"]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed building centrifuge-class")
    return LIB


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv, ptxas_v="--ptxas" in sys.argv)
