"""Build libsicp_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m simpleicp_b200._build [--force] [--verbose]

One object per translation unit (compiled in parallel), linked into
simpleicp_b200/libsicp_b200.so.  The library links the CUDA runtime statically and has no
dependency on torch or Python.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OBJ = PKG / "_build"
LIB = PKG / "libsicp_b200.so"
SOURCES = ["capi.cu", "batch.cu", "grid.cu", "nn.cu", "normals.cu", "reject_solve.cu", "transform.cu", "upload.cu", "io.cpp"]
CLI_SRC = PKG.parent / "cli" / "sicp_cli.cpp"
CLI_BIN = PKG / "sicp_cli"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
         "-Xptxas", "-v"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: libsicp_b200.so cannot be built")


def _digest() -> str:
    h = hashlib.sha256()
    for f in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.cpp")) +
                    [PKG.parent / "include" / "sicp_b200.h", CLI_SRC]):
        h.update(f.name.encode())
        h.update(f.read_bytes())
    h.update(" ".join(ARCH + FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    stamp = OBJ / "digest.txt"
    dig = _digest()
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == dig:
        return LIB
    nvcc = _nvcc()
    # several ranks / threads importing a fresh checkout must not write the same objects at once
    import fcntl

    with open(OBJ / "build.lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and LIB.exists() and stamp.exists() and stamp.read_text() == dig:
            return LIB  # another process built it while we waited
        return _build_locked(nvcc, dig, stamp, verbose)


def _build_locked(nvcc: str, dig: str, stamp: Path, verbose: bool) -> Path:

    def compile_one(src: str):
        obj = OBJ / (src.rsplit(".", 1)[0] + ".o")
        cmd = [nvcc, *ARCH, *FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, r

    objs = []
    with cf.ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        for src, obj, r in ex.map(compile_one, SOURCES):
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError(f"nvcc failed on {src}")
            (OBJ / (src.rsplit(".", 1)[0] + ".ptxas.txt")).write_text(r.stderr)
            if verbose:
                sys.stderr.write(r.stderr)
            objs.append(str(obj))
    cmd = [nvcc, *ARCH, "-shared", "-o", str(LIB), *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    # command-line front end with the reference CLI's flag set (c++/src/simpleicp-cli.cpp:15-35)
    cxx = shutil.which("g++") or "g++"
    cmd = [cxx, "-O2", "-std=c++17", "-I", str(PKG.parent / "include"), str(CLI_SRC), "-o", str(CLI_BIN),
           "-L", str(PKG), "-lsicp_b200", "-Wl,-rpath,$ORIGIN", "-lpthread", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("building sicp_cli failed")
    stamp.write_text(dig)
    return LIB


if __name__ == "__main__":
    lib = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(lib)
