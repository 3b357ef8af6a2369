"""Instruction inventory of one CUDA source file, per kernel and per source function (no GPU).

    python tools/sass_inventory.py simpleicp_b200/csrc/reject_solve.cu [--kernel k_rs_solve] [--top 12]

Compiles the file to a cubin with the package's nvcc flags (simpleicp_b200/_build.py), disassembles
it with `nvdisasm -gi` and attributes every instruction to the function whose body holds the source
line the line table gives it.  Functions of the project's sources are found by a scan for
`__device__` / `__global__` definitions.  An instruction of CUDA's own headers (a shuffle, a math
function) counts for the project function it was inlined into, under "name (header)".
A kernel's count includes the non-inlined device functions it calls (they are emitted into its
section).  Code that runs once per launch pays an instruction fetch per instruction, so these
counts are a first-order estimate of the cost of a cold first pass.
"""
from __future__ import annotations

import argparse
import functools
import bisect
import re
import subprocess
import sys
import tempfile
from collections import Counter
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from simpleicp_b200 import _build  # noqa: E402

_SECTION = re.compile(r"^\s*\.section\s+\.text\.(\S+?),")
_FILELINE = re.compile(r'//## File "([^"]+)", line (\d+)')
_INSN = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s+(\S.*?)\s*;")
_DEF = re.compile(r"^(?:template\s*<.*>\s*)?(?:static\s+)?(?:__\w+__\s+)")
_STRIP = re.compile(r"__launch_bounds__\s*\([^)]*\)|__align__\s*\([^)]*\)")


def function_starts(path: Path) -> tuple[list[int], list[str]]:
    """Start lines (1-based) and names of the device functions defined in a source file."""
    lines, names = [], []
    src = path.read_text().splitlines()
    i = 0
    while i < len(src):
        line = src[i]
        if _DEF.match(line) and ("__device__" in line or "__global__" in line):
            # the definition runs to the first '{' (a ';' first means a declaration)
            j, head = i, ""
            while j < len(src):
                head += " " + src[j]
                if "{" in src[j] or src[j].rstrip().endswith(";"):
                    break
                j += 1
            if "{" in src[j] or not src[j].rstrip().endswith(";"):
                m = re.search(r"([A-Za-z_]\w*)\s*\(", _STRIP.sub(" ", head.split("{")[0]))
                if m:
                    lines.append(i + 1)
                    names.append(m.group(1))
        i += 1
    return lines, names


def name_of(demangled: str) -> str:
    """Kernel name with its template arguments, without namespaces, return type and parameters."""
    d = re.sub(r"\(anonymous namespace\)::|<unnamed>::|\bsicp::|^void ", "", demangled)
    depth = 0
    for i, ch in enumerate(d):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return d[:i]
    return d


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("source", type=Path)
    ap.add_argument("--kernel", action="append", default=[],
                    help="substring of the kernels to report (default: all)")
    ap.add_argument("--top", type=int, default=12, help="functions listed per kernel")
    args = ap.parse_args()
    src = args.source.resolve()
    nvcc = _build._nvcc()
    nvdisasm = str(Path(nvcc).parent / "nvdisasm")
    cufilt = str(Path(nvcc).parent / "cu++filt")
    with tempfile.TemporaryDirectory() as tmp:
        cubin = Path(tmp) / "k.cubin"
        flags = [f for f in _build.FLAGS if f not in ("-Xcompiler", "-fPIC")]
        subprocess.run([nvcc, *_build.ARCH, *flags, "-cubin", str(src), "-o", str(cubin)], check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        sass = subprocess.run([nvdisasm, "-gi", "-c", str(cubin)], check=True, capture_output=True,
                              text=True).stdout

    starts: dict[str, tuple[list[int], list[str]]] = {}
    root = Path(__file__).resolve().parents[1]

    @functools.cache
    def ours(file: str) -> bool:
        return Path(file).resolve().is_relative_to(root)

    def owner(file: str, line: int) -> str:
        p = Path(file)
        if file not in starts:
            starts[file] = function_starts(p)
        ls, ns = starts[file]
        k = bisect.bisect_right(ls, line) - 1
        return f"{p.name}:{ns[k]}" if k >= 0 else p.name

    # -gi prints the inlining chain of an instruction as consecutive lines, innermost first
    kernels: dict[str, Counter] = {}
    cur, where, frames = None, "?", []
    for line in sass.splitlines():
        m = _SECTION.match(line)
        if m:
            cur = m.group(1)
            kernels[cur] = Counter()
            where, frames = "?", []
            continue
        m = _FILELINE.search(line)
        if m:
            frames.append((m.group(1), int(m.group(2))))
            continue
        m = _INSN.match(line)
        if cur is None or not m:
            continue
        if frames:
            mine = [f for f in frames if ours(f[0])]
            where = owner(*mine[0]) if mine else Path(frames[0][0]).name
            if mine and not ours(frames[0][0]):
                where += f" ({Path(frames[0][0]).name})"
            frames = []
        if m.group(1) != "NOP":  # (NOPs pad the section's end)
            kernels[cur][where] += 1

    mangled = list(kernels)
    demangled = subprocess.run([cufilt], input="\n".join(mangled), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    for mg, dm in zip(mangled, demangled):
        short = name_of(dm)
        if args.kernel and not any(k in dm for k in args.kernel):
            continue
        c = kernels[mg]
        print(f"{short:<40} {sum(c.values()):>6}")
        for name, n in c.most_common(args.top):
            print(f"    {n:>6}  {name}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
