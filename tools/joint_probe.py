"""Cost of the joint registration (sb.simpleicp_joint, sicp_register_joint) of a scan strip.

    python tools/joint_probe.py [--scans 256] [--points 100000] [--reps 5] [--out FILE]

Inputs: `scans` clouds of `points` points of the C3 surface (x in [2 i, 2 i + 26), y in [0, 30)),
each in its own frame (centred on its patch, then turned by up to 1 degree and moved by up to
0.3 m), start poses perturbed in that frame by 0.3 degrees and 5 cm, cloud 0 fixed; edges
(i, i + 1), (i, i + 2) and random loop closures (i, j) with 3 <= j - i <= 10, about 800 in all;
1000 correspondences, overlap filter 1 m.
Reported: the median over `reps` calls (after one warm-up call) of the wall time of the call and of
sicp_get_timings' device-event split per iteration -- match (match_ms), reject + edge blocks
(reject_solve_ms), joint solve + update (transform_ms) -- with the iteration count and the pose
error against the truth; the same edges through sb.simpleicp_edges under the linearised variant
(pairwise, the same rules without the joint solve);
and the NumPy restatement's time per iteration on the first 8 clouds and their edges.  The card
name and power limit are read in the same run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))

import simpleicp_b200 as sb  # noqa: E402
from oracle import joint_oracle as J  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def strip(n_scans, n_points, seed=7):
    rng = np.random.default_rng(seed)
    scans, truth, H0 = [], [], []
    for i in range(n_scans):
        x = rng.uniform(2.0 * i, 2.0 * i + 26.0, n_points)
        y = rng.uniform(0.0, 30.0, n_points)
        z = 0.05 * x + 0.03 * y + 2 * np.sin(2 * np.pi * x / 25) * np.cos(2 * np.pi * y / 40)
        P = np.column_stack((x, y, z + rng.normal(0, 0.01, n_points)))
        # the scan's frame: centred on its patch, then a small rigid transform
        T = J.rigid_from_x(np.concatenate((np.deg2rad(rng.uniform(-1, 1, 3)), rng.uniform(-0.3, 0.3, 3))))
        T[:3, 3] += (2.0 * i + 13.0, 15.0, 0.0)
        Ti = np.linalg.inv(T)
        scans.append(np.ascontiguousarray(P @ Ti[:3, :3].T + Ti[:3, 3]))
        truth.append(T)
        dH = J.rigid_from_x(np.concatenate((np.deg2rad(rng.normal(0, 0.3, 3)), rng.normal(0, 0.05, 3))))
        H0.append(T if i == 0 else T @ dH)
    edges = [(i, i + 1) for i in range(n_scans - 1)] + [(i, i + 2) for i in range(n_scans - 2)]
    seen = set(edges)
    while len(edges) < int(800 * n_scans / 256):
        i = int(rng.integers(0, n_scans - 3))
        j = i + int(rng.integers(3, 11))
        if j < n_scans and (i, j) not in seen:
            seen.add((i, j))
            edges.append((i, j))
    return scans, np.array(truth), np.array(H0), np.array(edges)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=256)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    scans, truth, H0, edges = strip(args.scans, args.points)
    kw = dict(correspondences=1000, max_overlap_distance=1.0)
    eng_key = 0
    runs = []
    for rep in range(args.reps + 1):
        t0 = time.perf_counter()
        res = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, on_error="nan", **kw)
        wall = time.perf_counter() - t0
        tm = sb.batch._BATCH_ENGINES[eng_key].timings()
        it = max(res.iterations, 1)
        runs.append({"wall_s": wall, "iterations": res.iterations, "converged": res.converged,
                     "match_ms_per_it": tm["match_ms"] / it, "reject_blocks_ms_per_it": tm["reject_solve_ms"] / it,
                     "solve_update_ms_per_it": tm["transform_ms"] / it,
                     "pose_err_max": float(np.abs(res.H - truth).max())})
    runs = runs[1:]
    med = {k: float(np.median([r[k] for r in runs])) for k in runs[0] if k != "converged"}
    # the same edges pairwise under the same (linearised) rules: the engine simpleicp_edges uses
    eng = sb.batch._BATCH_ENGINES[eng_key]
    eng.set_option("variant", 1)
    pair_wall = []
    try:
        for rep in range(args.reps + 1):
            t0 = time.perf_counter()
            sb.simpleicp_edges(scans, edges, batch_size=len(edges), on_error="nan", **kw)
            pair_wall.append(time.perf_counter() - t0)
    finally:
        eng.set_option("variant", 0)
    sub = [k for k, (a, b) in enumerate(edges) if b < 8]
    t0 = time.perf_counter()
    o = J.simpleicp_joint(scans[:8], edges[sub], fixed=(0,), H0=H0[:8], max_iterations=3,
                          max_overlap_distance=1.0)
    oracle_it = (time.perf_counter() - t0) / len(o.log)
    out = {"card": card(), "scans": args.scans, "points": args.points, "edges": int(len(edges)),
           "free_clouds": args.scans - 1, "joint_median": med, "joint_runs": runs,
           "edges_pairwise_wall_s_median": float(np.median(pair_wall[1:])),
           "oracle_s_per_iteration_8_clouds": oracle_it, "oracle_edges": len(sub)}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        Path(args.out).write_text(text)


if __name__ == "__main__":
    main()
