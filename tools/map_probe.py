"""Cost of registering many scans against one resident map (sb.Map, sicp_register_to_map).

    python tools/map_probe.py [--reps 3] [--out FILE]

Map: O.surface with about 10 M points over 1 km x 1 km.  Scans: 64 tiles of about 100 000 points
(100 m x 100 m) cut from a second realisation, each moved by a small rigid transform, with a
noisy prior and max_overlap_distance 1.0.  Reports the set_map time, the scans per second of
Map.register with the map resident, the overlap filter's share of the call and its bounded
searches (overlap_candidates), and, on a 2 M-point map at the same density (small enough for
the old route), the same job through simpleicp_batch with the map repeated for every scan; the
two routes alternate.  The card name and power limit are read in the same run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))

from oracle import simpleicp_oracle as O  # noqa: E402

import simpleicp_b200 as sb  # noqa: E402
from simpleicp_b200.simpleicp import _observed_in_radians  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def job(n_map, extent, n_scans=64, tile=100.0, seed=90_000):
    X = O.surface(n_map, seed, extent=extent)
    second = O.surface(n_map, seed + 1, extent=extent)
    rng = np.random.default_rng(seed)
    scans, rows = [], []
    for _ in range(n_scans):
        x0, y0 = rng.uniform(0, extent - tile, 2)
        m = (second[:, 0] >= x0) & (second[:, 0] < x0 + tile) & (second[:, 1] >= y0) & (second[:, 1] < y0 + tile)
        true = np.concatenate((rng.uniform(-0.5, 0.5, 3), rng.uniform(-0.3, 0.3, 3)))
        D = O.rbp_to_H(_observed_in_radians(true))
        scans.append(np.ascontiguousarray(O.transform_by_H(second[m], np.linalg.inv(D))))
        rows.append(true + np.concatenate((rng.normal(0, 0.05, 3), rng.normal(0, 0.03, 3))))
    return X, scans, np.array(rows)


def timed(fn):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    kw = dict(max_overlap_distance=1.0)
    rec = {"card": card()}

    # ---- 10 M-point map, resident
    X, scans, rows = job(10_000_000, 1000.0)
    rec["big"] = {"n_map": len(X), "n_scans": len(scans), "mean_scan": float(np.mean([len(s) for s in scans]))}
    t_set, m = timed(lambda: sb.Map(X))
    m.register(scans[:4], rbp_observed_values=rows[:4], on_error="nan", **kw)  # warm-up
    t_set2, _ = timed(lambda: m._engine.set_map(X))  # replacing the map: buffers already allocated
    calls = []
    for _ in range(a.reps):
        dt, table = timed(lambda: m.register(scans, rbp_observed_values=rows, on_error="nan", **kw))
        tm = m._engine.timings()
        calls.append({"s": dt, "overlap_ms": tm["overlap_ms"], "overlap_candidates": tm["overlap_candidates"],
                      "grid_mov_ms": tm["grid_mov_ms"], "normals_ms": tm["normals_ms"],
                      "loop_ms": tm["reject_solve_ms"]})
    best = min(calls, key=lambda c: c["s"])
    rec["big"].update({
        "set_map_s_first": t_set, "set_map_s": t_set2, "calls": calls,
        "scans_per_s": len(scans) / best["s"],
        "filter_share": best["overlap_ms"] / 1e3 / best["s"],
        "overlap_candidates": best["overlap_candidates"],
        "candidates_per_scan_and_map_point": best["overlap_candidates"] / (len(scans) * len(X)),
        "registered": int((table[:, 16] > 0).sum()),
    })
    m.close()
    del X, scans

    # ---- 2 M-point map: resident map against the map repeated for every pair, alternating
    X, scans, rows = job(2_000_000, 1000.0 * np.sqrt(0.2), seed=91_000)
    rec["small"] = {"n_map": len(X), "n_scans": len(scans), "map": [], "repeated": []}
    m = sb.Map(X)
    m.register(scans[:4], rbp_observed_values=rows[:4], on_error="nan", **kw)
    sb.simpleicp_batch([(X, s) for s in scans[:4]], rbp_observed_values=rows[:4], on_error="nan", **kw)
    for _ in range(a.reps):
        dt, t_map = timed(lambda: m.register(scans, rbp_observed_values=rows, on_error="nan", **kw))
        rec["small"]["map"].append(dt)
        dt, t_rep = timed(lambda: sb.simpleicp_batch([(X, s) for s in scans], rbp_observed_values=rows,
                                                     on_error="nan", **kw))
        rec["small"]["repeated"].append(dt)
    rec["small"]["same_table"] = bool(np.array_equal(t_map, t_rep, equal_nan=True))
    rec["small"]["scans_per_s_map"] = len(scans) / min(rec["small"]["map"])
    rec["small"]["scans_per_s_repeated"] = len(scans) / min(rec["small"]["repeated"])
    m.close()
    sb.close_engine_pool()

    print(json.dumps(rec, indent=1))
    if a.out:
        Path(a.out).write_text(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
