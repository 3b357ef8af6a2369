"""Cost of cloud-to-map distances (Map.distances, sicp_map_distances) against the host route.

    python tools/map_distances_probe.py [--reps 5] [--out FILE]

The set-up of tools/map_probe.py (DESIGN §6.2): a 10 M-point O.surface map over 1 km x 1 km and 64
scans of about 100 000 points, registered with max_overlap_distance 1.0; the registered scans are
then measured against the map with their H at max_distance 0.5 and 1.0, without and with
neighbors = 10.  Per case it reports the wall time of the raw C call from pinned inputs into pinned
outputs (host clock around a call that ends in a device synchronise; median and range over the
repetitions), the within points, and in a separate profiled call the device time of each kernel
(torch.profiler, CUDA activities).  The host route is Map.points(), a cKDTree over the map and a
query of the moved scans with distance_upper_bound (all cores), timed per step; its indices are
compared with the device's (np.array_equal).  The card name and power limit are read in the same
run."""
import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

from map_probe import card, job, timed  # noqa: E402

import simpleicp_b200 as sb  # noqa: E402


def pinned(a):
    import torch

    t = torch.empty(a.shape, dtype={np.float64: torch.float64, np.float32: torch.float32,
                                    np.int64: torch.int64}[a.dtype.type], pin_memory=True)
    t.numpy()[...] = a
    return t.numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from scipy.spatial import cKDTree

    rec = {"card": card()}
    X, scans, rows = job(10_000_000, 1000.0)
    m = sb.Map(X)
    kw = dict(max_overlap_distance=1.0, on_error="nan")
    m.register(scans[:4], rbp_observed_values=rows[:4], **kw)  # warm-up
    table, results = m.register(scans, rbp_observed_values=rows, full_output=True, **kw)
    ok = [i for i, r in enumerate(results) if r is not None]
    H = np.ascontiguousarray(table[ok, :16].reshape(-1, 4, 4))
    clouds = [pinned(scans[i]) for i in ok]
    moved = np.concatenate([results[i].X_mov_transformed for i in ok])
    n = [len(c) for c in clouds]
    rec.update(n_map=len(X), registered=len(ok), points=int(sum(n)))
    e = m._engine
    k_ = len(clouds)
    outs = {dt: [pinned(np.zeros(c, dt)) for c in n] for dt in (np.int64, np.float64, np.float32)}
    pd = [pinned(np.zeros(c)) for c in n]
    nw = np.zeros(k_, dtype=np.int64)
    ptrs = lambda L: (C.c_void_p * k_)(*[x.ctypes.data for x in L])  # noqa: E731

    def call(r, k):
        e._check(e._lib.sicp_map_distances(e._h, k_, ptrs(clouds), (C.c_int64 * k_)(*n), H.ctypes.data, r, k,
                                           ptrs(outs[np.int64]), ptrs(outs[np.float64]), ptrs(pd) if k else None,
                                           ptrs(outs[np.float32]) if k else None, nw.ctypes.data))

    tree_s = None
    for r in (0.5, 1.0):
        for k in (0, 10):
            name = f"r={r},k={k}"
            call(r, k)  # warm-up (buffers, modules)
            ts = []
            for _ in range(a.reps):
                dt, _ = timed(lambda: call(r, k))
                ts.append(dt)
            res = {"wall_s_median": float(np.median(ts)), "wall_s_range": [min(ts), max(ts)],
                   "within": int(nw.sum()), "fitness": float(nw.sum() / sum(n))}
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                call(r, k)
                torch.cuda.synchronize()
            kern = {}
            for ev in prof.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA:
                    kern[ev.name] = kern.get(ev.name, 0.0) + ev.device_time_total / 1e3
            res["device_ms"] = {kn: round(v, 3) for kn, v in sorted(kern.items(), key=lambda x: -x[1])}
            res["device_ms_total"] = round(sum(kern.values()), 3)
            rec[name] = res
        idx_dev = np.concatenate([x.copy() for x in outs[np.int64]])
        # the host route
        t0 = time.perf_counter()
        pts = m.points()
        t1 = time.perf_counter()
        if tree_s is None:
            tree = cKDTree(pts)
            tree_s = time.perf_counter() - t1
        t2 = time.perf_counter()
        _, ii = tree.query(moved, distance_upper_bound=r, workers=-1)
        t3 = time.perf_counter()
        ii = np.where(ii == len(pts), -1, ii)
        rec[f"host r={r}"] = {"points_s": t1 - t0, "tree_build_s": tree_s, "query_s": t3 - t2,
                              "total_s": (t1 - t0) + tree_s + (t3 - t2),
                              "same_indices": bool(np.array_equal(ii, idx_dev)),
                              "differing_indices": int((ii != idx_dev).sum())}
    m.close()
    print(json.dumps(rec, indent=1))
    if a.out:
        Path(a.out).write_text(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
