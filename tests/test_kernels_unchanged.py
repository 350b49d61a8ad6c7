"""The machine code of the kernels that existed before the inline-vector HNSW search is unchanged: every function in
tests/golden/kernels_sass.json (sm_90a, from the build before that change) must appear in the library's objects with the same SASS
and the same registers / stack / shared / local memory, after the anonymous-namespace hash (it depends on the source path) is
normalised away.  A change that alters one of these kernels on purpose regenerates the file:
    python tests/test_kernels_unchanged.py qdrant_b200/lib"""
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "kernels_sass.json")
LIB = os.path.join(ROOT, "qdrant_b200", "lib")
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
_ANON = re.compile(r"_GLOBAL__N__[0-9a-f]{8}_\d+_[A-Za-z0-9_]+?_cu_[0-9a-f]{8}")


def _norm(text: str) -> str:
    return _ANON.sub("_GLOBAL__N_", text)


def kernels(obj: str) -> dict:
    """{normalised function name: {"sass": sha256 of its normalised SASS, "res": its resource usage line}}"""
    sass = _norm(subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout)
    res = _norm(subprocess.run([CUOBJDUMP, "-res-usage", obj], capture_output=True, text=True, check=True).stdout)
    out, cur, buf = {}, None, []
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            if cur:
                out[cur] = {"sass": hashlib.sha256("\n".join(buf).encode()).hexdigest()}
            cur, buf = m.group(1), []
        elif cur:
            buf.append(line)
    if cur:
        out[cur] = {"sass": hashlib.sha256("\n".join(buf).encode()).hexdigest()}
    lines = res.splitlines()
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):$", line)
        if m and m.group(1) in out and i + 1 < len(lines):
            out[m.group(1)]["res"] = lines[i + 1].strip()
    return out


def test_pre_existing_kernels_compile_to_the_same_code():
    if not os.path.exists(CUOBJDUMP) and not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not installed")
    with open(GOLDEN) as f:
        golden = json.load(f)
    for obj, funcs in golden.items():
        path = os.path.join(LIB, obj)
        if not os.path.exists(path):
            pytest.skip(f"{path} not built (build() compiles the library)")
        got = kernels(path)
        for name, want in funcs.items():
            assert name in got, f"{obj}: {name} is gone"
            assert got[name] == want, f"{obj}: {name} changed: {got[name]} != {want}"


if __name__ == "__main__":
    d = sys.argv[1]
    data = {os.path.basename(p): kernels(os.path.join(d, p)) for p in sorted(os.listdir(d)) if p.endswith(".o")}
    with open(GOLDEN, "w") as f:
        json.dump({k: v for k, v in data.items() if v}, f, indent=0, sort_keys=True)
