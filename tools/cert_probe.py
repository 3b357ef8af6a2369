"""Diagnostics: how many queries of a C3 registration the match answers from its certificate
(nn.cu: MatchCert, DESIGN §3.2), iteration by iteration.  Not part of the product.

CPU part (no GPU needed): the oracle registers the C3 pair with a static tree, K queries,
min_change = 0 and 40 iterations.  From each iteration's moved queries and their exact first and
second neighbours (cKDTree) it replays the certificate rule with skin s: a search leaves
rho = (min(d2, d1 + s) - d1) / 2 around the query it searched (the scan's second-best or its
skinned skip limit, whichever is nearer), and a later query is certified while it stays inside.
Iteration 0 is a cold search and leaves no certificate.  Printed per iteration: the largest
query move since the previous iteration, the queries whose neighbour changed, and the predicted
certified count.

GPU part (--gpu): the same configuration through the staged API (sicp_iterate one iteration at
a time, sicp_debug_match_counts after each), printed next to the CPU prediction computed with the
device's skin kCertSkin * h.

    python tools/cert_probe.py [--points N] [--k K] [--iters 40] [--skin-cells 0.125] [--gpu]
"""
import argparse
import sys
from pathlib import Path

import numpy as np
from scipy.spatial import cKDTree

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import simpleicp_oracle as O  # noqa: E402


def cpu_prediction(X_fix, X_mov, K, iters, skin):
    tr = O.Trace()
    O.simpleicp(X_fix, X_mov, correspondences=K, min_change=0.0, max_iterations=iters, trace=tr,
                static_tree=True)
    tree = cKDTree(X_mov)
    P = X_fix[tr.idx_sel]
    rows, c, rho, prev_q, prev_nn = [], None, None, None, None
    for it, rec in enumerate(tr.iterations):
        q = O.transform_by_H(P, np.linalg.inv(rec.H_in))
        d, nn = tree.query(q, k=2)
        move = float(np.linalg.norm(q - prev_q, axis=1).max()) if prev_q is not None else float("nan")
        changed = int((nn[:, 0] != prev_nn).sum()) if prev_nn is not None else -1
        if it == 0:
            cert = np.zeros(len(q), dtype=bool)
        else:
            cert = np.zeros(len(q), dtype=bool) if c is None else np.linalg.norm(q - c, axis=1) < rho
        new_rho = 0.5 * (np.minimum(d[:, 1], d[:, 0] + skin) - d[:, 0])
        if it >= 1:  # the warm searches write certificates; a certified query keeps its own
            if c is None:
                c, rho = q.copy(), new_rho
            else:
                c[~cert], rho[~cert] = q[~cert], new_rho[~cert]
        rows.append((it, move, changed, int(cert.sum())))
        prev_q, prev_nn = q, nn[:, 0]
    return rows


def gpu_counts(X_fix, X_mov, K, iters):
    import simpleicp_b200 as sb
    from simpleicp_b200 import _capi

    with _capi.Engine() as e:
        e.set_clouds(X_fix, X_mov)
        e.set_selected(sb.pointcloud.subsample_indices(len(X_fix), K).astype(np.int64) if K < len(X_fix) else None)
        e.estimate_normals(10, download=False)
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        p = e.run_params(0.3, 0.0, 1000, lsq)
        counts = []
        for it in range(iters):
            e.iterate(p, x_in=np.zeros(6) if it == 0 else None)
            counts.append(e.match_counts())
        _, h, _ = e.grid_params("mov")
    return counts, h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=100_000)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--skin-cells", type=float, default=0.125, help="nn.cu: kCertSkin")
    ap.add_argument("--skin-m", type=float, default=0.02, help="skin of the CPU part without --gpu (m)")
    ap.add_argument("--gpu", action="store_true")
    a = ap.parse_args()
    X_fix, X_mov, _ = O.c3_pair(a.points)
    gpu, skin = None, a.skin_m
    if a.gpu:
        gpu, h = gpu_counts(X_fix, X_mov, a.k, a.iters)
        skin = a.skin_cells * h
        print(f"movable grid cell h = {h:.4f} m, skin = {skin:.4f} m")
    rows = cpu_prediction(X_fix, X_mov, a.k, a.iters, skin)
    print(f"{'it':>3} {'max move (m)':>13} {'nn changed':>10} {'certified (CPU)':>15}" + (f" {'certified (GPU)':>15}" if gpu else ""))
    for it, move, changed, cert in rows:
        line = f"{it:>3} {move:>13.3g} {changed:>10} {cert:>15}"
        if gpu:
            line += f" {gpu[it]:>15}"
        print(line)


if __name__ == "__main__":
    main()
