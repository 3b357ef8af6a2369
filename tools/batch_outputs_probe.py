"""Cost of full_output (sicp_get_batch_outputs) on the batched engine and on the resident map.

    python tools/batch_outputs_probe.py [--reps 5] [--out FILE]

C5 batch: 64 pairs of 100 000 points in pinned memory (bench.make_c5_pairs), one
simpleicp_batch call.  Map: the 10 M-point map and 64 scans of tools/map_probe.py, one
Map.register call with max_overlap_distance 1.0.  Each job alternates the default call and the
full_output=True call (same arguments) after warm-ups and reports the median wall time of each.
Then one getter call on a plain engine is traced with torch.profiler: device time of the
segmented transform, the residual compaction and the copies, by kind (the clouds come back
into pinned NumPy arrays, 24 bytes per movable point).  The card name and power limit are
read in the same run."""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

import simpleicp_b200 as sb  # noqa: E402
from bench import make_c5_pairs  # noqa: E402
from map_probe import card, job  # noqa: E402
from simpleicp_b200 import _capi  # noqa: E402
from simpleicp_b200.simpleicp import _observed_in_radians  # noqa: E402


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def alternate(plain, full, reps):
    plain(), full()  # warm-ups: buffers, pinned pools
    a, b = [], []
    for _ in range(reps):
        dt, t_plain = timed(plain)
        a.append(dt)
        dt, (t_full, results) = timed(full)
        b.append(dt)
    return {"default_s": statistics.median(a), "full_output_s": statistics.median(b), "default_all": a,
            "full_output_all": b, "same_table": bool(np.array_equal(t_plain, t_full, equal_nan=True)),
            "results": sum(r is not None for r in results)}


def getter_trace(e, register):
    """Device time per stage of one getter call on engine `e` after `register()` (a call of `e`
    returning the PairResult array), by torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    res = register()
    outs = None
    for _ in range(2):  # the second call is the traced one (pinned pools warm)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            outs = e.batch_outputs(res)
            wall = time.perf_counter() - t0
    stages = {}
    for k in prof.key_averages():
        us = getattr(k, "device_time_total", None) or getattr(k, "cuda_time_total", 0.0)
        name = k.key
        for tag in ("k_transform_pairs", "k_batch_residuals", "Memcpy DtoH", "Memcpy HtoD", "Memcpy DtoD"):
            if tag in name:
                stages[tag] = stages.get(tag, 0.0) + us / 1e3
    bytes_xyz = sum(o[0].nbytes for o in outs if o is not None)
    return {"wall_ms": wall * 1e3, "device_ms": stages, "cloud_bytes": bytes_xyz,
            "cloud_GBps_by_DtoH": bytes_xyz / (stages.get("Memcpy DtoH", np.nan) * 1e-3) / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rec = {"card": card()}

    # ---- C5 batch
    pairs = make_c5_pairs(range(64), 100_000, pinned=True)
    rec["c5"] = alternate(lambda: sb.simpleicp_batch(pairs, on_error="nan", batch_size=64),
                          lambda: sb.simpleicp_batch(pairs, on_error="nan", batch_size=64, full_output=True), a.reps)
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
        rec["c5"]["getter"] = getter_trace(e, lambda: e.register_batch(pairs, 1000, 10, params))
    sb.close_engine_pool()
    del pairs
    print(json.dumps(rec, indent=1), flush=True)

    # ---- 10 M-point map, 64 scans
    X, scans, rows = job(10_000_000, 1000.0)
    kw = dict(max_overlap_distance=1.0, rbp_observed_values=rows, on_error="nan")
    with sb.Map(X) as m:
        rec["map"] = alternate(lambda: m.register(scans, **kw), lambda: m.register(scans, full_output=True, **kw),
                               a.reps)
        e = m._engine
        params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
        rad = np.array([_observed_in_radians(r) for r in rows])
        rec["map"]["getter"] = getter_trace(e, lambda: e.register_to_map(scans, 1000, 10, params, 1.0, rad))
    rec["map"]["movable_points"] = int(sum(len(s) for s in scans))

    print(json.dumps(rec, indent=1))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
