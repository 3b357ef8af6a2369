"""Cost of registering a scan sequence's edges with shared clouds (sb.simpleicp_edges,
sicp_register_pairs) against the same pairs expanded (sb.simpleicp_batch, sicp_register_batch).

    python tools/edges_probe.py [--reps 2] [--scans 256] [--out FILE]

Inputs: a sequence of 256 scans of 100 000 points, scan i = the movable cloud of C5 pair i
(synthetic.c5_pair: a 30 m x 30 m patch of the surface moved by a small rigid transform), with
the edges (i, i + 1) and (i, i + 2) in sequence order: 509 in all, 64 per library call.  Both
routes run with and without mov_neighbors = 10, alternating.  Reported per run: the wall time of the whole call, the
sums over its library calls of sicp_get_timings' upload_ms (the upload of the clouds that are fixed
in some pair; the movable-only clouds cross PCIe on the copy stream while the fixed side computes),
grid_fix_ms + grid_mov_ms, mov_normals_ms and reject_solve_ms (the loop), the clouds uploaded, and
whether the two tables are equal.  The card name and power limit are read in the same run."""
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
from simpleicp_b200 import _capi, synthetic  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


STAGES = ("upload_ms", "grid_fix_ms", "grid_mov_ms", "mov_normals_ms", "reject_solve_ms")
_LOG = []


def _spy(name):
    """Engine.<name> recording, after every library call, its timings and the clouds it uploaded."""
    orig = getattr(_capi.Engine, name)

    def call(self, *a, **kw):
        out = orig(self, *a, **kw)
        tm = self.timings()
        clouds = sum(c is not None for c in a[0]) if name == "register_pairs" else 2 * len(a[0])
        _LOG.append({**{k: tm[k] for k in STAGES}, "clouds": clouds})
        return out

    setattr(_capi.Engine, name, call)


def run(fn):
    import torch

    _LOG.clear()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    table = fn()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    rec = {"s": dt, "calls": len(_LOG), "clouds_uploaded": sum(c["clouds"] for c in _LOG)}
    rec.update({k: sum(c[k] for c in _LOG) for k in STAGES})
    return rec, table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--scans", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.scans
    scans = [synthetic.c5_pair(i, 100_000, n)[1] for i in range(n)]
    # in sequence order, as an odometry front end produces them: (0, 1), (0, 2), (1, 2), (1, 3), ...
    edges = np.array([(i, j) for i in range(n) for j in (i + 1, i + 2) if j < n])
    pairs = [(scans[f], scans[m]) for f, m in edges]
    _spy("register_pairs")
    _spy("register_batch")
    rec = {"card": card(), "n_scans": n, "n_edges": len(edges), "batch_size": 64}
    for k_mov in (0, 10):
        kw = dict(mov_neighbors=k_mov) if k_mov else {}
        sb.simpleicp_edges(scans, edges[:64], on_error="nan", **kw)  # warm-up (buffer growth)
        sb.simpleicp_batch(pairs[:64], on_error="nan", **kw)
        runs = {"edges": [], "batch": []}
        for _ in range(a.reps):
            r_e, t_e = run(lambda: sb.simpleicp_edges(scans, edges, on_error="nan", **kw))
            r_b, t_b = run(lambda: sb.simpleicp_batch(pairs, on_error="nan", **kw))
            runs["edges"].append(r_e)
            runs["batch"].append(r_b)
        runs["same_table"] = bool(np.array_equal(t_e, t_b, equal_nan=True))
        runs["registered"] = int((t_e[:, 16] > 0).sum())
        runs["speedup"] = min(r["s"] for r in runs["batch"]) / min(r["s"] for r in runs["edges"])
        rec[f"mov_neighbors={k_mov}"] = runs
    sb.close_engine_pool()
    print(json.dumps(rec, indent=1))
    if a.out:
        Path(a.out).write_text(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
