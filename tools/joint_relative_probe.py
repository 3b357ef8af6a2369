"""Measure relative pose observations in sicp_register_joint_relative (DESIGN.md §6.13).

    python tools/joint_relative_probe.py [--config 256x100000x800] [--long 1024x5000x3000] [--reps N] [--out FILE]

1. Cost, on the strip of tests/test_gpu_joint.py (256 clouds x 100 000 points, 800 edges, F = 255):
   under each solve (dense, sparse), without observations and with 255 odometry links (i, i + 1)
   (the truth plus 0.02 degrees and 2 cm), the four calls alternated: sicp_timings'
   reject_solve_ms (k_joint_reject and k_joint_relative) and transform_ms (the solve) per
   iteration, medians over the repeats; then one call of each under torch.profiler for the device
   time per launch of k_joint_relative and of the solve kernel.
2. Accuracy, on a long strip (1024 clouds, cloud 0 fixed, the sparse solve): the same call without
   observations and with odometry (i, i + 1) from the truth plus 0.01 degrees and 1 cm, weighted for
   rows of 1 cm; RMS position and rotation error of the free clouds against the truth.
The card's name and power limit are read in the same run.  One JSON line per measurement on stdout
(and in FILE with --out).
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch
from scipy.spatial.transform import Rotation

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tests"))

from simpleicp_b200 import _capi  # noqa: E402
from simpleicp_b200._capi import SicpError  # noqa: E402
from test_gpu_joint import strip  # noqa: E402
from joint_sparse_probe import card  # noqa: E402


def odometry(truth, seed, rot_deg, pos_m, row_m):
    """(i, i + 1) for every cloud: T_i^-1 T_(i+1) of the truth moved by seeded noise, weighted for rows
    of row_m metres."""
    rng = np.random.default_rng(seed)
    n = len(truth)
    pairs = np.array([(i, i + 1) for i in range(n - 1)], dtype=np.int64)
    Z = []
    for a, b in pairs:
        E = np.eye(4)
        E[:3, :3] = Rotation.from_rotvec(np.deg2rad(rng.normal(0, rot_deg, 3))).as_matrix()
        E[:3, 3] = rng.normal(0, pos_m, 3)
        Z.append(np.linalg.inv(truth[a]) @ truth[b] @ E)
    W = np.tile([row_m ** 2 / np.deg2rad(rot_deg) ** 2] * 3 + [row_m ** 2 / pos_m ** 2] * 3, (n - 1, 1))
    return pairs, np.array(Z), W


def errors(H, truth, free):
    pos = np.linalg.norm(H[:, :3, 3] - truth[:, :3, 3], axis=1)[free]
    rot = np.linalg.norm(Rotation.from_matrix(H[:, :3, :3] @ np.transpose(truth[:, :3, :3], (0, 2, 1))).as_rotvec(),
                         axis=1)[free]
    return float(np.sqrt(np.mean(pos ** 2))), float(np.rad2deg(np.sqrt(np.mean(rot ** 2)))), float(pos.max())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="256x100000x800")
    ap.add_argument("--long", default="1024x5000x3000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-iterations", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("joint_relative_probe needs a CUDA device")
    info = card()
    lines = []

    def emit(line):
        line = {**line, **info}
        print(json.dumps(line), flush=True)
        lines.append(line)

    eng = _capi.Engine(0)
    lsq = eng.lsq_params((0.0,) * 6, (0.0,) * 6, [0.0] * 6, 1)
    params = eng.run_params(0.3, 1.0, args.max_iterations, lsq)

    # ---- 1. cost on the 256-cloud strip
    n, points, n_edges = (int(v) for v in args.config.split("x"))
    scans, truth, H0, edges = strip(n, points, n_edges)
    rel = odometry(truth, 41, 0.02, 0.02, 0.01)
    fixed = np.zeros(n, dtype=bool)
    fixed[0] = True
    runs = [(s, r) for s in (0, 1) for r in (False, True)]

    def call(solver, with_rel):
        eng.set_option("joint_solver", solver)
        H, out = eng.register_joint(scans, edges, fixed, H0, 1000, 10, params, 1.0, None, None,
                                    *(rel if with_rel else ()))
        return out[0].iterations, eng.timings()

    for r in runs:
        call(*r)  # warm-up of every shape
    rows = {r: [] for r in runs}
    for _ in range(args.reps):
        for r in runs:
            its, t = call(*r)
            rows[r].append((t["reject_solve_ms"] / its, t["transform_ms"] / its, its))
    from torch.profiler import ProfilerActivity, profile
    for r in runs:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(*r)
            torch.cuda.synchronize()
        k = {}
        for ev in prof.key_averages():
            for name in ("k_joint_relative", "k_joint_sparse_solve", "k_joint_solve", "k_joint_reject"):
                if name in ev.key:
                    k[name] = {"calls": ev.count, "device_us_per_call": ev.device_time_total / ev.count}
                    break
        a = np.array(rows[r])
        emit({"clouds": n, "points": points, "edges": int(len(edges)), "F": n - 1, "solver": ["dense", "sparse"][r[0]],
              "observations": len(rel[0]) if r[1] else 0, "iterations": int(a[0, 2]),
              "reject_and_relative_ms_per_it": float(np.median(a[:, 0])), "solve_ms_per_it": float(np.median(a[:, 1])),
              "kernels": k})

    # ---- 2. accuracy on a long strip, sparse solve
    n, points, n_edges = (int(v) for v in args.long.split("x"))
    scans, truth, H0, edges = strip(n, points, n_edges, seed=12)
    rel = odometry(truth, 43, 0.01, 0.01, 0.01)
    fixed = np.zeros(n, dtype=bool)
    fixed[0] = True
    free = ~fixed
    eng.set_option("joint_solver", 1)
    for with_rel in (False, True):
        t0 = time.perf_counter()
        line = {"long_strip": n, "points": points, "edges": int(len(edges)),
                "observations": len(rel[0]) if with_rel else 0,
                "odometry_rot_deg": 0.01, "odometry_pos_m": 0.01}
        try:
            H, out = eng.register_joint(scans, edges, fixed, H0, 1000, 10, params, 1.0, None, None,
                                        *(rel if with_rel else ()))
            pos, rot, mx = errors(H, truth, free)
            st = {int(k): int(v) for k, v in zip(*np.unique([o.status for o in out], return_counts=True))}
            line.update(status=0, edge_statuses=st, iterations=int(out[0].iterations), converged=bool(out[0].converged),
                        pos_rms_m=pos, rot_rms_deg=rot, max_pos_m=mx)
        except SicpError as ex:
            line.update(status=int(ex.code), error=str(ex))
        line["call_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        p0, r0, m0 = errors(H0, truth, free)
        line.update(start_pos_rms_m=p0, start_rot_rms_deg=r0)
        emit(line)
    eng.set_option("joint_solver", 0)
    eng.close()
    if args.out:
        Path(args.out).write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
