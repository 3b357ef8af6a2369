"""Measure sicp_overlap_graph on the strip of tests/test_gpu_joint.py (DESIGN.md §6.10).

    python tools/overlap_graph_probe.py [--configs 1024x100000 4096x100000 ...] [--out FILE]

For each configuration (clouds x points per cloud) and stride 1 and 10, at r = 1.0 under the generator's perturbed poses: one
warm-up call, then 5 timed calls; the median of sicp_timings (upload_ms, grid_fix_ms, overlap_ms)
and of CUDA events around the call; the reported pairs; the candidate directions and bounded
searches of the two culls restated with the clouds' bounding boxes (the library culls with its grid
boxes, up to one cell larger, so these are lower bounds); searches per second over overlap_ms.  The
card's name and power limit are read in the same run.  One JSON line per configuration on stdout (and
in FILE with --out); a call the library refuses (e.g. more grid cells than one grid build holds) is
recorded with its message.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tests"))

from simpleicp_b200 import _capi  # noqa: E402
from test_gpu_joint import strip  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def restated_culls(scans, H, r, s):
    """(candidate directions, bounded searches) of the two culls with bounding boxes, on the GPU."""
    dev = torch.device("cuda")
    lo = np.array([X.min(0) for X in scans])
    hi = np.array([X.max(0) for X in scans])
    corners = np.array([[(hi if k & (1 << a) else lo)[:, a] for a in range(3)] for k in range(8)])  # 8 x 3 x N
    corners = np.transpose(corners, (2, 0, 1))  # N x 8 x 3
    world = np.einsum("nij,nkj->nki", H[:, :3, :3], corners) + H[:, None, :3, 3]
    wlo, whi = world.min(1) - r / 2, world.max(1) + r / 2
    wlo_t, whi_t = torch.tensor(wlo, device=dev), torch.tensor(whi, device=dev)
    meet = ((wlo_t[:, None, :] <= whi_t[None, :, :]) & (wlo_t[None, :, :] <= whi_t[:, None, :])).all(-1)
    meet.fill_diagonal_(False)
    directions = searches = 0
    Hinv = np.linalg.inv(H)
    for a in range(len(scans)):
        bs = torch.nonzero(meet[a]).flatten().cpu().numpy()
        if len(bs) == 0:
            continue
        T = Hinv[a] @ H[bs]  # a <- b
        box = np.einsum("nij,nkj->nki", T[:, :3, :3], corners[bs]) + T[:, None, :3, 3]
        blo = torch.tensor(box.min(1) - r, device=dev)
        bhi = torch.tensor(box.max(1) + r, device=dev)
        P = torch.tensor(scans[a][::s], device=dev)
        inside = ((P[None] >= blo[:, None]) & (P[None] <= bhi[:, None])).all(-1).sum(1)
        directions += int((inside > 0).sum())
        searches += int(inside.sum())
    return directions, searches


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["1024x100000", "4096x100000", "256x100000", "1024x20000",
                                                      "4096x5000"])
    ap.add_argument("--strides", type=int, nargs="+", default=[1, 10])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("overlap_graph_probe needs a CUDA device")
    info = card()
    eng = _capi.Engine(0)
    r = 1.0
    lines = []
    for cfg in args.configs:
        n, points = (int(v) for v in cfg.split("x"))
        scans, truth, H0, _ = strip(n, points, 1)
        for s in args.strides:
            base = {"clouds": n, "points": points, "r": r, "stride": s, **info}
            try:
                eng.overlap_graph(scans, H0, max_distance=r, stride=s, cap=0)  # warm-up
            except _capi.SicpError as e:
                line = {**base, "refused": e.message}
                print(json.dumps(line), flush=True)
                lines.append(line)
                continue
            rows = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                total, _, _ = eng.overlap_graph(scans, H0, max_distance=r, stride=s, cap=0)
                e1.record()
                e1.synchronize()
                t = eng.timings()
                rows.append((e0.elapsed_time(e1), t["upload_ms"], t["grid_fix_ms"], t["overlap_ms"], total))
            med = np.median(np.array(rows, dtype=np.float64), axis=0)
            directions, searches = restated_culls(scans, H0, r, s)
            line = {**base, "call_ms": med[0], "upload_ms": med[1], "grid_fix_ms": med[2], "overlap_ms": med[3],
                    "pairs": int(rows[-1][4]), "directions_bbox": directions, "searches_bbox": searches,
                    "searches_per_s": searches / (med[3] * 1e-3)}
            print(json.dumps(line), flush=True)
            lines.append(line)
        del scans
    eng.close()
    if args.out:
        Path(args.out).write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
