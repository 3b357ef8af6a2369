"""Cost of the movable-normals estimate (sicp_register_params.mov_neighbors) on the GPU.

    python tools/mov_normals_probe.py [--out FILE.json] [--reps 7]

C3 (1 M <-> 1 M points, 100 000 correspondences): sicp_register with and without
mov_neighbors = 10, median end-to-end time over `reps` calls after two warm-ups, the device time of
the estimate (timings mov_normals_ms) and both runs' iteration and kept counts; the estimate's time
for several bounds of its neighbour scratch (option "normals_scratch_mb", which sets the queries per launch).
C5 (64 pairs of 100 000 points, 1000 correspondences): batch pairs/s with and without.
The card's name and power limit are read in the same process.  A summary is printed; --out also
writes the full record (every timing and kept count) as JSON.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import simpleicp_b200 as sb  # noqa: E402
from simpleicp_b200 import _capi  # noqa: E402
from simpleicp_b200.synthetic import c3_pair, c5_pair  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": q[0] if q else "unavailable"}


def c3(reps: int) -> dict:
    import torch

    X_fix, X_mov, _ = c3_pair()
    out = {}
    with _capi.Engine() as e:
        for label, k in (("without", None), ("mov_neighbors_10", 10)):
            times, r = [], None
            for i in range(reps + 2):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                r = sb.register(X_fix, X_mov, correspondences=100_000, want_normals=False, engine=e,
                                mov_neighbors=k)
                torch.cuda.synchronize()
                if i >= 2:
                    times.append((time.perf_counter() - t0) * 1e3)
            out[label] = {"e2e_ms_median": float(np.median(times)), "e2e_ms_all": times,
                          "mov_normals_ms": r.timings["mov_normals_ms"], "normals_ms": r.timings["normals_ms"],
                          "iterations": r.iterations, "kept": [rec["n_kept"] for rec in r.records]}
        sweep = {}
        for mb in (4, 16, 64, 256):  # at k = 10 and 10^6 queries: 10, 3, 1 and 1 launches
            e.reset_options()
            e.set_option("normals_scratch_mb", mb)
            ms = []
            for i in range(reps + 1):
                sb.register(X_fix, X_mov, correspondences=100_000, want_normals=False, engine=e, mov_neighbors=10,
                            max_iterations=1)
                if i >= 1:
                    ms.append(e.timings()["mov_normals_ms"])
            sweep[str(mb)] = {"mov_normals_ms_median": float(np.median(ms)), "all": ms,
                              "queries_per_launch_k10": (mb << 20) // 40}
        out["scratch_sweep"] = sweep
    return out


def c5(reps: int) -> dict:
    import torch

    pairs = [c5_pair(i)[:2] for i in range(64)]
    pinned = []
    for Xf, Xm in pairs:
        a = _capi.pinned_empty(Xf.shape, np.float64)
        b = _capi.pinned_empty(Xm.shape, np.float64)
        a[:] = Xf
        b[:] = Xm
        pinned.append((a, b))
    out = {}
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
        for label, k in (("without", 0), ("mov_neighbors_10", 10)):
            times, res = [], None
            for i in range(reps + 2):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = e.register_batch(pinned, 1000, 10, params, mov_neighbors=k)
                torch.cuda.synchronize()
                if i >= 2:
                    times.append(time.perf_counter() - t0)
            out[label] = {"pairs_per_s_median": 64 / float(np.median(times)),
                          "mov_normals_ms": e.timings()["mov_normals_ms"],
                          "iterations_mean": float(np.mean([r.iterations for r in res])),
                          "n_kept_mean": float(np.mean([r.n_kept for r in res])),
                          "status": sorted({int(r.status) for r in res})}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="write the full record as JSON to this file")
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    rec = {"card": card(), "c3": c3(a.reps), "c5": c5(a.reps)}
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rec, indent=1))
    print(json.dumps({"card": rec["card"],
                      "c3": {k: {kk: v[kk] for kk in v if kk not in ("e2e_ms_all", "kept")}
                             for k, v in rec["c3"].items() if k != "scratch_sweep"},
                      "c3_scratch_mb": {k: v["mov_normals_ms_median"] for k, v in rec["c3"]["scratch_sweep"].items()},
                      "c5": rec["c5"]}, indent=1))


if __name__ == "__main__":
    main()
