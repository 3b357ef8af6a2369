"""Cost of shrinking a resident map on the device (Map.crop, Map.thin; sicp_map_crop, sicp_map_thin).

    python tools/map_crop_probe.py [--reps 5] [--out FILE]

The set-up of tools/map_probe.py and map_insert_probe.py (DESIGN §6.2, §6.4): a 10 M-point
O.surface map over 1 km x 1 km and 64 scans of about 100 000 points with noisy priors,
max_overlap_distance 1.0.  The scans are registered; the positions of those that register are the
centroids of their moved points (the scans are tiles of the map's frame, so H's translation is not
a sensor position here).  It reports, per case, the wall time of the call (host clock around a call
that ends in a device synchronise; the map is reset before each repetition; median and range) and
the points removed, for
  - a crop around the registered scans' positions at radius 100 m and 200 m,
  - a thin at v = h and v = 4 h, h = sqrt(3 A / n) the map grid's first cell-size estimate;
the host route (Map.points(), the NumPy rule, Map(...)), whose points must equal the device's; and
Map.register of the 64 scans on the full map and on the cropped map, alternating the two in one
loop.  The card name and power limit are read in the same run."""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

from map_probe import card, job, timed  # noqa: E402

import simpleicp_b200 as sb  # noqa: E402


def crop_on_host(M, centers, r):
    """The crop rule in NumPy, one centre at a time: (dx dx + dy dy) + dz dz < r * r for any centre."""
    keep = np.zeros(len(M), dtype=bool)
    for c in centers:
        d = M - c
        keep |= (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] < r * r
    return M[keep]


def thin_on_host(M, v):
    """The thin rule in NumPy: the first point of every voxel key floor(p / v), in map order."""
    _, first = np.unique(np.floor(M / v) + 0.0, axis=0, return_index=True)
    return M[np.sort(first)]


def stats(ts):
    return {"median_ms": 1e3 * float(np.median(ts)), "min_ms": 1e3 * float(np.min(ts)),
            "max_ms": 1e3 * float(np.max(ts))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    kw = dict(max_overlap_distance=1.0, on_error="nan")
    rec = {"card": card()}
    X, scans, rows = job(10_000_000, 1000.0)
    ext = X.max(axis=0) - X.min(axis=0)
    h = float(np.sqrt(3.0 * ext[0] * ext[1] / len(X)))
    rec.update(n_map=len(X), n_scans=len(scans), scan_points=int(sum(len(s) for s in scans)), cell_size=h)
    m = sb.Map(X)
    m.register(scans[:4], rbp_observed_values=rows[:4], **kw)  # warm-up
    table, results = m.register(scans, rbp_observed_values=rows, full_output=True, **kw)
    ok = [i for i, r in enumerate(results) if r is not None]
    centers = np.array([results[i].X_mov_transformed.mean(axis=0) for i in ok])
    rec["registered"] = len(ok)
    m0 = sb.Map(X)  # the full map, registered against alternately with the cropped one
    m0.register(scans, rbp_observed_values=rows, **kw)

    def reset():
        m._engine.set_map(X)
        m.n_points = m._engine.n_map

    reset()
    m.crop(centers[:2], radius=50.0)  # warm-up of both paths
    reset()
    m.thin(voxel_size=4 * h)
    cases = [("crop r=100", lambda: m.crop(centers, radius=100.0), lambda P: crop_on_host(P, centers, 100.0)),
             ("crop r=200", lambda: m.crop(centers, radius=200.0), lambda P: crop_on_host(P, centers, 200.0)),
             ("thin v=h", lambda: m.thin(voxel_size=h), lambda P: thin_on_host(P, h)),
             ("thin v=4h", lambda: m.thin(voxel_size=4 * h), lambda P: thin_on_host(P, 4 * h))]
    for name, call, host in cases:
        r = {"call_s": []}
        for _ in range(a.reps):
            reset()
            dt, removed = timed(call)
            r["call_s"].append(dt)
        r.update(stats(r["call_s"]))
        r["removed"], r["n_after"] = int(removed), int(m.n_points)
        shrunk = m.points()
        if name.startswith("crop"):
            m.register(scans, rbp_observed_values=rows, **kw)  # warm-up on the cropped map
            r["register_s_full"], r["register_s_cropped"] = [], []
            for _ in range(a.reps):
                dt, t_full = timed(lambda: m0.register(scans, rbp_observed_values=rows, **kw))
                r["register_s_full"].append(dt)
                dt, t_crop = timed(lambda: m.register(scans, rbp_observed_values=rows, **kw))
                r["register_s_cropped"].append(dt)
            r["registered_full"] = int((t_full[:, 16] > 0).sum())
            r["registered_cropped"] = int((t_crop[:, 16] > 0).sum())
        # the host route from the full map: read it back, apply the rule on the host, upload a new map
        reset()
        dt, fresh = timed(lambda: sb.Map(host(m.points())))
        r["host_route_s"] = dt
        r["same_points"] = bool(np.array_equal(fresh.points(), shrunk))
        fresh.close()
        rec[name] = r
        print(name, json.dumps({k: v for k, v in r.items() if not isinstance(v, list)}), flush=True)
    m.close()
    m0.close()
    print(json.dumps(rec, indent=1))
    if a.out:
        Path(a.out).write_text(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
