"""Cost of growing a resident map with registered scans (Map.insert, sicp_map_insert).

    python tools/map_insert_probe.py [--reps 5] [--out FILE]

The set-up of tools/map_probe.py (DESIGN §6.2): a 10 M-point O.surface map over 1 km x 1 km and
64 scans of about 100 000 points with noisy priors, max_overlap_distance 1.0.  The scans are
registered, then inserted with their H at a voxel size v equal to the map grid's cell size as the
builder first estimates it (sqrt(3 A / n), A the map's x-y extent) and at 4 v.  Per voxel size it
reports the insert's wall time (host clock around a call that ends in a device synchronise; the
map is reset before each repetition), the points added, Map.register of the 64 scans on a second
Map of the original points and on the grown map, alternating the two in one loop, and the same
job done on the host (Map.points(), NumPy thinning to the same rule, Map(...)), whose points must
equal the device's.  For the registration times it also reports the mean iterations of both tables
and the first-pass cell plan of the map grid (first_cell_plan) for both point sets.  The card name and power limit are read in the same run."""
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


def thin_on_host(M, clouds, v):
    """The insert rule in NumPy: the first finite point of every voxel key floor(p / v) that no
    map point has, appended in order."""
    C = np.concatenate(clouds)
    fin = np.flatnonzero(np.isfinite(C).all(axis=1))
    with np.errstate(over="ignore", invalid="ignore"):
        K = np.floor(np.concatenate([M, C[fin]]) / v) + 0.0
    _, first = np.unique(K, axis=0, return_index=True)
    return np.concatenate([M, C[fin[np.sort(first[first >= len(M)]) - len(M)]]])


def first_cell_plan(P, occ=3.0, cap=1 << 25):
    """The cell size and dims grid_build (grid.cu) picks for one cloud under the batch policy
    (grid_plan.h: first_cell_plan) before it refines from the measured occupancy, which it skips
    when the cell cap binds (as for these maps)."""
    ext = P.max(axis=0) - P.min(axis=0)
    e = np.sort(ext)
    emax = max(e[2], 1e-12)
    h = max(np.sqrt(occ * max(e[2] * max(e[1], 1e-3 * emax), 1e-300) / len(P)), emax * 1e-6)
    bound = False
    while True:
        d = [max(1, int(np.floor(x / h)) + 1) for x in ext]
        if d[0] * d[1] * d[2] <= min(cap, max(4096, 32 * len(P))):
            return {"h": h, "dims": d, "cap_binds": bound, "extent": ext.tolist()}
        h *= 1.26
        bound = True


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
    H = table[ok, :16].reshape(-1, 4, 4)
    clouds = [scans[i] for i in ok]
    moved = [results[i].X_mov_transformed for i in ok]
    rec["registered"] = len(ok)
    m0 = sb.Map(X)  # the original map, registered against alternately with the grown one
    m0.register(scans, rbp_observed_values=rows, **kw)
    m.insert(clouds[:2], H[:2], voxel_size=h)  # warm-up of the insert path
    for name, v in (("v=h", h), ("v=4h", 4 * h)):
        r = {"voxel_size": v, "insert_s": []}
        for _ in range(a.reps):
            m._engine.set_map(X)
            m.n_points = m._engine.n_map
            dt, added = timed(lambda: m.insert(clouds, H, voxel_size=v))
            r["insert_s"].append(dt)
        r["added"] = int(added.sum())
        m.register(scans, rbp_observed_values=rows, **kw)  # warm-up on the grown map
        r["register_s_original"], r["register_s_grown"] = [], []
        for _ in range(a.reps):
            dt, t_orig = timed(lambda: m0.register(scans, rbp_observed_values=rows, **kw))
            r["register_s_original"].append(dt)
            dt, t_grown = timed(lambda: m.register(scans, rbp_observed_values=rows, **kw))
            r["register_s_grown"].append(dt)
        r["iterations_original"] = float(t_orig[t_orig[:, 16] > 0, 16].mean())
        r["iterations_grown"] = float(t_grown[t_grown[:, 16] > 0, 16].mean())
        grown = m.points()
        r["cell_plan_original"], r["cell_plan_grown"] = first_cell_plan(X), first_cell_plan(grown)
        # the host route from the original map: read it back, thin on the host, upload a new map
        m._engine.set_map(X)
        m.n_points = m._engine.n_map
        dt, fresh = timed(lambda: sb.Map(thin_on_host(m.points(), moved, v)))
        r["host_route_s"] = dt
        r["same_points"] = bool(np.array_equal(fresh.points(), grown))
        fresh.close()
        rec[name] = r
    m.close()
    m0.close()
    print(json.dumps(rec, indent=1))
    if a.out:
        Path(a.out).write_text(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
