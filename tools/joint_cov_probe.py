"""Cost of the a-posteriori covariances of a joint registration (sicp_get_joint_covariances) on
tools/joint_probe.py's scan strip: 256 scans, about 800 edges, F = 255 free clouds, 1530 unknowns.

    python tools/joint_cov_probe.py [--scans 256] [--points 100000] [--reps 5] [--out FILE]

Per rep: one sb.simpleicp_joint call, then the first covariance request (the one that computes).
Reported, as medians over the reps after one warm-up: the wall time of that request (launches,
device work and the download of the blocks), and from torch.profiler (CUPTI device timestamps) the
device time of each covariance kernel and of the registration's k_joint_solve per iteration, which
the covariances are compared against.  The card name and power limit are read in the same run."""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

import simpleicp_b200 as sb  # noqa: E402
from joint_probe import card, strip  # noqa: E402

KERNELS = ("k_joint_cov_ss", "k_joint_inv", "k_joint_cov_cloud", "k_joint_cov_edge", "k_joint_solve")


def device_ms(prof):
    """Summed device time (ms) and launch count per kernel of KERNELS."""
    out = {k: [0.0, 0] for k in KERNELS}
    for ev in prof.events():
        name = ev.name
        for k in KERNELS:
            if k + "(" in name or name.endswith(k):
                t = getattr(ev, "device_time", None)
                if t is None:
                    t = ev.cuda_time
                out[k][0] += t / 1000.0
                out[k][1] += 1
    return out


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=256)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    scans, truth, H0, edges = strip(args.scans, args.points)
    kw = dict(correspondences=1000, max_overlap_distance=1.0)
    runs = []
    for rep in range(args.reps + 1):
        res = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, on_error="nan", **kw)
        eng = sb.batch._BATCH_ENGINES[0]
        t0 = time.perf_counter()
        cov, ecov, s0 = eng.joint_covariances(len(scans), len(edges))
        wall = time.perf_counter() - t0
        runs.append({"get_wall_ms": wall * 1e3, "s0": s0, "iterations": res.iterations})
    runs = runs[1:]
    # device times of one more registration and its covariances
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        res = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, on_error="nan", **kw)
        eng = sb.batch._BATCH_ENGINES[0]
        eng.joint_covariances(len(scans), len(edges))
        torch.cuda.synchronize()
    dev = device_ms(prof)
    cov_ms = sum(dev[k][0] for k in KERNELS[:4])
    solve = dev["k_joint_solve"]
    out = {"card": card(), "scans": args.scans, "points": args.points, "edges": int(len(edges)),
           "free_clouds": args.scans - 1, "unknowns": 6 * (args.scans - 1),
           "get_wall_ms_median": float(np.median([r["get_wall_ms"] for r in runs])),
           "cov_kernels_device_ms": {k: dev[k][0] for k in KERNELS[:4]}, "cov_device_ms": cov_ms,
           "joint_solve_device_ms_per_iteration": solve[0] / max(solve[1], 1),
           "joint_solve_launches": solve[1], "iterations": res.iterations, "runs": runs}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        Path(args.out).write_text(text)


if __name__ == "__main__":
    main()
