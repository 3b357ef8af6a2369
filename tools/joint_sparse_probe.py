"""Measure sicp_register_joint under the dense and the sparse solve (DESIGN.md §6.11) on the strip of
tests/test_gpu_joint.py.

    python tools/joint_sparse_probe.py [--configs 256x100000x800 1024x20000x3200 ...] [--reps N]
                                       [--profile] [--out FILE]

Configurations are clouds x points per cloud x edges.  The 256-cloud strip (F = 255) runs under both
solvers, alternated call by call; larger ones only under the sparse solve.  Every shape is warmed up
first; then per call the host clock around it (the call ends in a device synchronise) and
sicp_timings' match_ms, reject_solve_ms and transform_ms (match; reject + edge blocks; solve +
update) per iteration.  Medians over the repeats, with min and max.  The plan's supernodes, tree
depth and factor bytes come from csrc/joint_plan.h compiled with g++ over the same edges.  The
card's name and power limit are read in the same run.  --profile instead times the solve kernels
with torch.profiler (one call per configuration after the warm-up).  One JSON line per
configuration and solver on stdout (and in FILE with --out).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tests"))

from simpleicp_b200 import _capi  # noqa: E402
from test_gpu_joint import strip  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def plan_stats(F: int, pairs: np.ndarray) -> dict:
    """n_super, depth and factor bytes of joint_plan.h's plan over the free-free pairs."""
    with tempfile.TemporaryDirectory() as d:
        so = Path(d) / "libjoint_plan_host.so"
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", str(REPO / "tests" / "native" /
                        "joint_plan_host.cpp"), "-o", str(so)], check=True)
        lib = C.CDLL(str(so))
        lib.joint_plan_build.restype = C.c_longlong
        p = np.ascontiguousarray(pairs.astype(np.int32))
        n = lib.joint_plan_build(F, len(p), p.ctypes.data_as(C.c_void_p), None, C.c_longlong(0))
        buf = np.zeros(n, dtype=np.int64)
        lib.joint_plan_build(F, len(p), p.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p), C.c_longlong(n))
    return {"supernodes": int(buf[1]), "depth": int(buf[2]), "factor_bytes": int(8 * buf[-1])}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["256x100000x800", "1024x20000x3200", "4096x5000x12800"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-iterations", type=int, default=30)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("joint_sparse_probe needs a CUDA device")
    info = card()
    eng = _capi.Engine(0)
    lsq = eng.lsq_params((0.0,) * 6, (0.0,) * 6, [0.0] * 6, 1)
    params = eng.run_params(0.3, 1.0, args.max_iterations, lsq)
    lines = []
    for cfg in args.configs:
        n, points, n_edges = (int(v) for v in cfg.split("x"))
        scans, truth, H0, edges = strip(n, points, n_edges)
        fixed = np.zeros(n, dtype=bool)
        fixed[0] = True
        solvers = [0, 1] if n - 1 <= 256 else [1]
        free = edges[(edges[:, 0] > 0) & (edges[:, 1] > 0)] - 1
        stats = plan_stats(n - 1, free)

        def call(solver):
            eng.set_option("joint_solver", solver)
            t0 = time.perf_counter()
            H, out = eng.register_joint(scans, edges, fixed, H0, 1000, 10, params, 1.0)
            wall = (time.perf_counter() - t0) * 1e3
            return wall, out[0].iterations, eng.timings()

        try:
            for s in solvers:
                call(s)  # warm-up of every shape
        except _capi.SicpError as e:
            line = {"clouds": n, "points": points, "edges": int(len(edges)), "F": n - 1, "refused": e.message,
                    **stats, **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
            continue
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            for s in solvers:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    _, its, _ = call(s)
                    torch.cuda.synchronize()
                k = {}
                for ev in prof.key_averages():
                    if "k_joint" in ev.key:
                        name = ev.key.split("k_joint")[1].split("(")[0].split("E")[0]
                        k["k_joint" + name] = {"calls": ev.count, "device_ms_per_call": ev.device_time_total / ev.count / 1e3}
                line = {"clouds": n, "points": points, "edges": int(len(edges)), "solver": ["dense", "sparse"][s],
                        "iterations": its, "kernels": k, **info}
                print(json.dumps(line), flush=True)
                lines.append(line)
            continue
        rows = {s: [] for s in solvers}
        for _ in range(args.reps):
            for s in solvers:  # alternated
                wall, its, t = call(s)
                rows[s].append((wall, t["match_ms"] / its, t["reject_solve_ms"] / its, t["transform_ms"] / its, its))
        for s in solvers:
            a = np.array(rows[s])
            stat = lambda j: {"median": float(np.median(a[:, j])), "min": float(a[:, j].min()), "max": float(a[:, j].max())}
            line = {"clouds": n, "points": points, "edges": int(len(edges)), "F": n - 1, "solver": ["dense", "sparse"][s],
                    "iterations": int(a[0, 4]), "call_ms": stat(0), "match_ms_per_it": stat(1),
                    "reject_ms_per_it": stat(2), "solve_ms_per_it": stat(3), **stats, **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
        del scans
    eng.set_option("joint_solver", 0)
    eng.close()
    if args.out:
        Path(args.out).write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
