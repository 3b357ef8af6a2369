"""Measure the cost of pose priors in sicp_register_joint_priors (DESIGN.md §6.12) on the strip of
tests/test_gpu_joint.py (256 clouds x 100 000 points, 800 edges, F = 255).

    python tools/joint_prior_probe.py [--config 256x100000x800] [--reps N] [--out FILE]

Under each solve (dense, sparse), without priors and with a prior on every free cloud (truth plus
0.02 degrees and 3 cm), the four calls alternated: sicp_timings' reject_solve_ms (which holds
k_joint_reject and k_joint_prior) and transform_ms (the solve) per iteration, medians over the
repeats.  Then one call of each under torch.profiler for the device time per launch of
k_joint_prior and of the solve kernel.  The card's name and power limit are read in the same run.
One JSON line per solve and prior setting on stdout (and in FILE with --out).
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tests"))

from simpleicp_b200 import _capi  # noqa: E402
from test_gpu_joint import strip  # noqa: E402
from joint_sparse_probe import card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="256x100000x800")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-iterations", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("joint_prior_probe needs a CUDA device")
    info = card()
    n, points, n_edges = (int(v) for v in args.config.split("x"))
    scans, truth, H0, edges = strip(n, points, n_edges)
    rng = np.random.default_rng(41)
    P = np.array(truth)
    for k in range(n):
        w = np.deg2rad(rng.normal(0, 0.02, 3))
        th = np.linalg.norm(w)
        K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / max(th, 1e-300)
        P[k, :3, :3] = (np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K) @ P[k, :3, :3]
        P[k, :3, 3] += rng.normal(0, 0.03, 3)
    W = np.tile([0.01 ** 2 / np.deg2rad(0.02) ** 2] * 3 + [0.01 ** 2 / 0.03 ** 2] * 3, (n, 1))
    fixed = np.zeros(n, dtype=bool)
    fixed[0] = True
    eng = _capi.Engine(0)
    lsq = eng.lsq_params((0.0,) * 6, (0.0,) * 6, [0.0] * 6, 1)
    params = eng.run_params(0.3, 1.0, args.max_iterations, lsq)
    runs = [(s, pr) for s in (0, 1) for pr in (False, True)]

    def call(solver, priors):
        eng.set_option("joint_solver", solver)
        H, out = eng.register_joint(scans, edges, fixed, H0, 1000, 10, params, 1.0, P if priors else None,
                                    W if priors else None)
        return out[0].iterations, eng.timings()

    for r in runs:
        call(*r)  # warm-up of every shape
    rows = {r: [] for r in runs}
    for _ in range(args.reps):
        for r in runs:
            its, t = call(*r)
            rows[r].append((t["reject_solve_ms"] / its, t["transform_ms"] / its, its))
    kern = {}
    from torch.profiler import ProfilerActivity, profile
    for r in runs:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(*r)
            torch.cuda.synchronize()
        k = {}
        for ev in prof.key_averages():
            for name in ("k_joint_prior", "k_joint_sparse_solve", "k_joint_solve", "k_joint_reject"):
                if name in ev.key:
                    k[name] = {"calls": ev.count, "device_us_per_call": ev.device_time_total / ev.count}
                    break
        kern[r] = k
    lines = []
    for r in runs:
        a = np.array(rows[r])
        line = {"clouds": n, "points": points, "edges": int(len(edges)), "F": n - 1,
                "solver": ["dense", "sparse"][r[0]], "priors": r[1], "iterations": int(a[0, 2]),
                "reject_and_prior_ms_per_it": float(np.median(a[:, 0])), "solve_ms_per_it": float(np.median(a[:, 1])),
                "kernels": kern[r], **info}
        print(json.dumps(line), flush=True)
        lines.append(line)
    eng.set_option("joint_solver", 0)
    eng.close()
    if args.out:
        Path(args.out).write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
