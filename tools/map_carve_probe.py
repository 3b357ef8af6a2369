"""Cost of carving a resident map on the device (Map.carve, sicp_map_carve).

    python tools/map_carve_probe.py [--reps 5] [--out FILE]

The map of tools/map_probe.py (DESIGN §6.2, §6.4, §6.6): 10 M O.surface points over 1 km x 1 km.
64 scans: each sensor stands 2 m above the surface at a random position, and its scan's
endpoints are the points of a second realisation of the terrain (synthetic.surface) within 50 m
of it horizontally; the sensor is the scan's origin.  It reports the wall time of one carve of all
64 scans (host clock around a call that ends in a device synchronise; the map is reset before
each repetition; median and range) at radius 0.05 m, margin 0.5 m and min_passes 2, and the
points removed.  The NumPy rule is timed on a subsample of rays against the whole map and
extrapolated to all rays (labelled as such).  The card name and power limit are read in the
same run."""
import argparse
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
from simpleicp_b200 import synthetic  # noqa: E402


def passes_on_host(M, o, P, r, margin):
    """The carve rule in NumPy, one ray at a time against every map point."""
    out = np.zeros(len(M), dtype=np.int64)
    u = [M[:, i] for i in range(3)]
    for p in P:
        d = p - o
        L2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
        if not (L2 > 0 and np.isfinite(L2)):
            continue
        L = np.sqrt(L2)
        ux, uy, uz = u[0] - o[0], u[1] - o[1], u[2] - o[2]
        s = ((ux * d[0] + uy * d[1]) + uz * d[2]) / L
        e2 = ((ux * ux + uy * uy) + uz * uz) - s * s
        out += (s > 0) & (s < L - margin) & (e2 < r * r)
    return out


def scans_of(T, n_scans, radius, height, seed):
    """n_scans sensors `height` above the terrain T and, per sensor, T's points within `radius`."""
    rng = np.random.default_rng(seed)
    lo, hi = T.min(axis=0), T.max(axis=0)
    cell = radius
    key = np.floor((T[:, :2] - lo[:2]) / cell).astype(np.int64)
    nx = int(key[:, 0].max()) + 1
    order = np.argsort(key[:, 1] * nx + key[:, 0], kind="stable")
    flat = (key[:, 1] * nx + key[:, 0])[order]
    scans, origins = [], []
    for _ in range(n_scans):
        s = np.array([rng.uniform(lo[0] + radius, hi[0] - radius), rng.uniform(lo[1] + radius, hi[1] - radius)])
        c = np.floor((s - lo[:2]) / cell).astype(np.int64)
        idx = []
        for gy in range(c[1] - 1, c[1] + 2):
            a, b = np.searchsorted(flat, [gy * nx + c[0] - 1, gy * nx + c[0] + 2])
            idx.append(order[a:b])
        cand = T[np.concatenate(idx)]
        near = cand[np.linalg.norm(cand[:, :2] - s, axis=1) < radius]
        ground = near[np.argmin(np.linalg.norm(near[:, :2] - s, axis=1)), 2]
        scans.append(np.ascontiguousarray(near))
        origins.append([s[0], s[1], ground + height])
    return scans, np.array(origins)


def stats(ts):
    return {"median_ms": 1e3 * float(np.median(ts)), "min_ms": 1e3 * float(np.min(ts)),
            "max_ms": 1e3 * float(np.max(ts))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    r, margin, k = 0.05, 0.5, 2
    rec = {"card": card(), "radius": r, "margin": margin, "min_passes": k}
    X, _, _ = job(10_000_000, 1000.0, n_scans=0)
    T = synthetic.surface(10_000_000, 91_000, extent=1000.0)
    scans, origins = scans_of(T, 64, 50.0, 2.0, 92_000)
    rec.update(n_map=len(X), n_scans=len(scans), rays=int(sum(len(s) for s in scans)))
    m = sb.Map(X)

    def reset():
        m._engine.set_map(X)
        m.n_points = m._engine.n_map

    reset()
    m.carve(scans[:2], origins=origins[:2], radius=r, margin=margin, min_passes=k)  # warm-up
    ts = []
    for _ in range(a.reps):
        reset()
        dt, (removed, passes) = timed(lambda: m.carve(scans, origins=origins, radius=r, margin=margin,
                                                      min_passes=k, return_passes=True))
        ts.append(dt)
    row = stats(ts)
    row.update(removed=int(removed), removed_min_passes_1=int((passes >= 1).sum()), max_passes=int(passes.max()))
    rec["carve"] = row
    print("carve", json.dumps(row), flush=True)
    # the NumPy rule: a subsample of rays against the whole map, extrapolated to every ray
    rng = np.random.default_rng(93_000)
    sub = [(i, j) for i, j in zip(rng.integers(0, len(scans), 4), rng.integers(0, 1000, 4))]
    t0 = time.perf_counter()
    for i, j in sub:
        passes_on_host(X, origins[i], scans[i][j % len(scans[i])][None], r, margin)
    per_ray = (time.perf_counter() - t0) / len(sub)
    rec["numpy_rule_s_per_ray"] = per_ray
    rec["numpy_rule_s_all_rays_extrapolated"] = per_ray * rec["rays"]
    m.close()
    print(json.dumps(rec, indent=1))
    if a.out:
        Path(a.out).write_text(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
