"""Builds libqdrant_b200.so in-tree with nvcc for sm_90a / H100 (no torch, no cmake).

    python -m qdrant_b200.build [--force] [--verbose]

The .so and the objects are build products (git-ignored).
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "lib")
OUT = os.path.join(OUT_DIR, "libqdrant_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]   # H100: wgmma, TMA, clusters

FLAGS = [
    *ARCH,
    "-O3", "-lineinfo", "-std=c++17",
    "--fmad=false",            # never contract a*b+c: every FMA in the kernels is an explicit __fmaf_rn
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-O3",
    "-Xptxas", "-v",
    "-shared", "-cudart", "static",
]


def sources() -> list[str]:
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + [
        os.path.join(HERE, "..", "include", "qb200.h"), os.path.abspath(__file__)] + glob.glob(os.path.join(HERE, "host", "*"))   # build.py: flags
    if not os.path.exists(os.path.join(OUT_DIR, "host_selftest")):
        return True
    return any(os.path.getmtime(d) > t for d in deps)


def build_variant(name: str, defines: list[str]) -> str:
    """Experiment builds: libqdrant_b200_<name>.so with extra -D flags (build-time knobs), selected at run time with QB_LIB_PATH.
    Not part of the product build."""
    out = os.path.join(OUT_DIR, f"libqdrant_b200_{name}.so")
    vdir = os.path.join(OUT_DIR, "variant_" + name)
    os.makedirs(vdir, exist_ok=True)
    objs, procs = [], []
    for src in sources():
        obj = os.path.join(vdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC] + [f for f in FLAGS if f not in ("-shared",)] + defines + ["-c", src, "-o", obj]
        cmd = [c for i, c in enumerate(cmd) if c != "-cudart" and (i == 0 or cmd[i - 1] != "-cudart")]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        o, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(o)
            raise RuntimeError("nvcc failed")
    r = subprocess.run([NVCC, *ARCH, "-shared", "-cudart", "static", "-o", out] + objs + ["-lpthread", "-ldl", "-lrt"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return OUT
    os.makedirs(OUT_DIR, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(OUT_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC] + [f for f in FLAGS if f not in ("-shared",)] + ["-c", src, "-o", obj]
        # remove the -cudart pair for compile-only steps
        cmd = [c for i, c in enumerate(cmd) if c != "-cudart" and (i == 0 or cmd[i - 1] != "-cudart")]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {os.path.basename(src)}\n{out}")
        failed |= p.returncode != 0
    with open(os.path.join(OUT_DIR, "build.log"), "w") as f:
        f.write("\n".join(log))
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("nvcc failed")
    if verbose:
        print("\n".join(log))
    link = [NVCC, *ARCH, "-shared", "-cudart", "static", "-o", OUT] + objs + ["-lpthread", "-ldl", "-lrt"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    # C++ host-side mirror self-test (drives the .so through qdrant_b200/host/qdrant_b200.hpp)
    host = os.path.join(HERE, "host")
    cmd = ["g++", "-std=c++17", "-O2", "-I", host, os.path.join(host, "host_selftest.cpp"), "-L", OUT_DIR, "-lqdrant_b200",
           "-Wl,-rpath,$ORIGIN", "-o", os.path.join(OUT_DIR, "host_selftest")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("host_selftest build failed")
    return OUT


if __name__ == "__main__":
    if "--variant" in sys.argv:
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], [a for a in sys.argv[i + 2:] if a.startswith("-D")]))
    else:
        print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
