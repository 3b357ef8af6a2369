"""Measure sicp_get_joint_selected_covariances after a sparse joint call (DESIGN.md §6.14).

    python tools/joint_sparse_cov_probe.py [--problems strip256 strip1024 strip4096_priors block64]
                                           [--reps N] [--out FILE]

Problems: §6.9's strip (256 clouds x 100 000 points, F = 255), the 1 024 x 20 000 strip (F = 1 023),
the 4 096 x 5 000 strip held by priors (F = 4 095, fixed=(), started from the priors) and the 64 x 64
block of tests/test_gpu_joint_graphs.py (F = 4 095).  Each runs one sparse call with
max_iterations=1 (the request's cost does not depend on the iterations run) and then:
  - the whole request, by the host clock around it (it ends in a copy to the host), on `reps`
    fresh calls; the first request after each call computes, later ones copy the cache;
  - the device time of every kernel of one request and of the call's k_joint_sparse_solve, with
    torch.profiler, in a run of its own.
Medians with min and max.  The card's name and power limit are read in the same run.  One JSON
line per problem on stdout (and in FILE with --out).
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tests"))

from simpleicp_b200 import _capi  # noqa: E402
from test_gpu_joint import strip  # noqa: E402
from test_gpu_joint_graphs import _block  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def _noisy(truth, seed, rot_deg, pos_m):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    R = Rotation.from_rotvec(np.deg2rad(rng.normal(0, rot_deg, (len(truth), 3)))).as_matrix()
    P = np.array(truth, dtype=np.float64)
    P[:, :3, :3] = R @ P[:, :3, :3]
    P[:, :3, 3] += rng.normal(0, pos_m, (len(truth), 3))
    return P


def problem(name):
    """scans, edges, is_fixed, H0, prior poses, prior weights"""
    P = W = None
    if name == "strip256":
        scans, truth, H0, edges = strip(256, 100_000, 800)
    elif name == "strip1024":
        scans, truth, H0, edges = strip(1024, 20_000, 3_200)
    elif name == "strip4096_priors":
        scans, truth, H0, edges = strip(4096, 5_000, 12_800)
        P = _noisy(truth, 41, 0.03, 0.05)
        W = np.tile([0.01 ** 2 / np.deg2rad(0.03) ** 2] * 3 + [0.01 ** 2 / 0.05 ** 2] * 3, (4096, 1))
        H0 = P.copy()
    elif name == "block64":
        scans, truth, H0, edges = _block(64)
    else:
        raise KeyError(name)
    fixed = np.zeros(len(scans), dtype=bool)
    if P is None:
        fixed[0] = True
    return scans, np.asarray(edges), fixed, H0, P, W


def _kernels(prof):
    k = {}
    for ev in prof.key_averages():
        if "k_joint" in ev.key:
            name = "k_joint" + ev.key.split("k_joint")[1].split("(")[0].split("E")[0]
            k[name] = {"calls": ev.count, "device_ms": round(ev.device_time_total / 1e3, 4)}
    return k


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--problems", nargs="+", default=["strip256", "strip1024", "strip4096_priors", "block64"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("joint_sparse_cov_probe needs a CUDA device")
    from torch.profiler import ProfilerActivity, profile
    info = card()
    eng = _capi.Engine(0)
    lsq = eng.lsq_params((0.0,) * 6, (0.0,) * 6, [0.0] * 6, 1)
    params = eng.run_params(0.3, 1.0, 1, lsq)
    eng.set_option("joint_solver", 1)
    lines = []
    for name in args.problems:
        scans, edges, fixed, H0, P, W = problem(name)

        def call():
            eng.register_joint(scans, edges, fixed, H0, 1000, 10, params, 1.0, P, W)
            torch.cuda.synchronize()

        call()  # warm-up of every shape, the request's included
        eng.joint_selected_covariances(len(scans), len(edges))
        walls, cached = [], []
        for _ in range(args.reps):
            call()
            t0 = time.perf_counter()
            eng.joint_selected_covariances(len(scans), len(edges))
            walls.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            cov, ecov, s0 = eng.joint_selected_covariances(len(scans), len(edges))
            cached.append((time.perf_counter() - t0) * 1e3)
        call()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.joint_selected_covariances(len(scans), len(edges))
            torch.cuda.synchronize()
        req = _kernels(prof)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
        solve = _kernels(prof).get("k_joint_sparse_solve", {})
        line = {"problem": name, "clouds": len(scans), "edges": int(len(edges)), "F": int((~fixed).sum()),
                "request_ms_median": round(float(np.median(walls)), 3), "request_ms_min": round(min(walls), 3),
                "request_ms_max": round(max(walls), 3), "cached_request_ms": round(float(np.median(cached)), 3),
                "request_kernels": req, "k_joint_sparse_solve_ms": solve.get("device_ms"), "s0": s0,
                "finite": bool(np.isfinite(cov[~fixed]).all() and np.isfinite(ecov).all()), **info}
        print(json.dumps(line), flush=True)
        lines.append(line)
    eng.set_option("joint_solver", 0)
    eng.close()
    if args.out:
        Path(args.out).write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
