"""The a-posteriori covariances of a joint registration (DESIGN.md §6.9) restated in NumPy on top of
the joint restatement (oracle/joint_oracle.py), for the tests.

The covariances come from the final iteration of a finished oracle run `res`.  The oracle's steps
are deterministic, so the same call stopped one iteration earlier gives the poses that iteration
started from.  From those poses this module repeats the final iteration: for every edge the match,
the median / MAD rejection and the kept rows A xi = l in frame a, with the selection and normals of
`res`.  It then assembles the joint matrix Nbig over the edges with >= 6 kept rows and solves it.
That gives s0^2 = sum r^2 / (sum n_e - 6 F), r = A xi - l.  The maps J_c, G_a and G_b at the final
poses are applied to s0^2 Nbig^-1.  The unknowns x_c are taken about the world origin, as in the
oracle, so J_c = [[I, 0], [-[o_c]x, I]]."""
from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np
from scipy import spatial

from oracle import joint_oracle as J
from oracle.linearized_oracle import mad_upper, median_upper


@dataclass
class FinalIteration:
    H: np.ndarray = None       # (n_clouds, 4, 4) poses after the repeated final iteration
    A: List[np.ndarray] = field(default_factory=list)   # per edge: the kept rows in frame a
    l: List[np.ndarray] = field(default_factory=list)
    xi: List[np.ndarray] = field(default_factory=list)  # per edge: the increment in frame a (None: no part)
    N: np.ndarray = None       # the joint matrix Nbig
    slot: Dict[int, int] = field(default_factory=dict)  # free cloud -> its block of Nbig
    s0: float = float("nan")
    cov: np.ndarray = None     # (n_clouds, 6, 6) of (omega_c, d o_c)
    edge_cov: np.ndarray = None  # (n_edges, 6, 6) of (alpha_e, d q_e) in frame a


def lever(P: np.ndarray, d: np.ndarray) -> np.ndarray:
    """[[P, 0], [-P [d]x, P]]"""
    M = np.zeros((6, 6))
    M[:3, :3] = P
    M[3:, 3:] = P
    M[3:, :3] = -P @ J.skew(d)
    return M


def final_iteration(clouds, edges, res, fixed=(0,), H0=None, min_planarity: float = 0.3, **kw) -> FinalIteration:
    """The final iteration of `res` = J.simpleicp_joint(clouds, edges, fixed=fixed, H0=H0,
    min_planarity=min_planarity, **kw), and its covariances."""
    edges = np.asarray(edges, dtype=np.int64)
    n_clouds = len(clouds)
    nrm = {e: (res.normals[e], res.planarity[e]) for e in range(len(edges))}
    kw = {k: v for k, v in kw.items() if k not in ("max_iterations", "normals")}
    pre = J.simpleicp_joint(clouds, edges, fixed=fixed, H0=H0, min_planarity=min_planarity,
                            max_iterations=len(res.log) - 1, normals=nrm, **kw)
    T = [np.array(h) for h in pre.H]
    used = np.zeros(n_clouds, dtype=bool)
    used[edges.ravel()] = True
    is_fixed = np.zeros(n_clouds, dtype=bool)
    is_fixed[list(fixed)] = True
    slot = {c: k for k, c in enumerate(c for c in range(n_clouds) if used[c] and not is_fixed[c])}
    F = len(slot)
    out = FinalIteration(slot=slot)
    rows = []
    for e, (a, b) in enumerate(edges):
        R = np.linalg.inv(T[a]) @ T[b]
        Xb = np.asarray(clouds[b], dtype=np.float64)
        P1 = np.asarray(clouds[a], dtype=np.float64)[res.idx_fix[e]]
        Ri = np.linalg.inv(R)
        _, nn = spatial.cKDTree(Xb).query(P1 @ Ri[:3, :3].T + Ri[:3, 3], k=1, workers=-1)
        P2 = Xb[nn] @ R[:3, :3].T + R[:3, 3]
        n = np.asarray(res.normals[e], dtype=np.float64)
        d = np.einsum("ij,ij->i", P2 - P1, n)
        med = median_upper(d)
        sig = 1.4826 * mad_upper(d)
        keep = ~((np.abs(d - med) > 3.0 * sig) | (res.planarity[e] < min_planarity))
        p1, p2, nk = P1[keep], P2[keep], n[keep]
        A = np.empty((p1.shape[0], 6))
        A[:, 0] = -p2[:, 2] * nk[:, 1] + p2[:, 1] * nk[:, 2]
        A[:, 1] = p2[:, 2] * nk[:, 0] - p2[:, 0] * nk[:, 2]
        A[:, 2] = -p2[:, 1] * nk[:, 0] + p2[:, 0] * nk[:, 1]
        A[:, 3:6] = nk
        rows.append((A, np.einsum("ij,ij->i", nk, p1 - p2), J.ad_world_to_frame(T[a])))
    Nbig = np.zeros((6 * F, 6 * F))
    gbig = np.zeros(6 * F)
    for e, (a, b) in enumerate(edges):
        A, l, Ad = rows[e]
        if A.shape[0] < 6:
            continue
        N = Ad.T @ (A.T @ A) @ Ad
        g = Ad.T @ (A.T @ l)
        for c, s in ((a, -1.0), (b, 1.0)):
            if c in slot:
                i = 6 * slot[c]
                Nbig[i:i + 6, i:i + 6] += N
                gbig[i:i + 6] += s * g
        if a in slot and b in slot:
            i, j = 6 * slot[a], 6 * slot[b]
            Nbig[i:i + 6, j:j + 6] -= N
            Nbig[j:j + 6, i:i + 6] -= N
    xs = np.linalg.solve(Nbig, gbig)
    x = {c: xs[6 * k:6 * k + 6] for c, k in slot.items()}
    ss, m = 0.0, 0
    for e, (a, b) in enumerate(edges):
        A, l, Ad = rows[e]
        out.A.append(A)
        out.l.append(l)
        if A.shape[0] < 6:
            out.xi.append(None)
            continue
        xi = Ad @ (x.get(b, np.zeros(6)) - x.get(a, np.zeros(6)))
        out.xi.append(xi)
        r = A @ xi - l
        ss += float(r @ r)
        m += A.shape[0]
    for c in slot:
        T[c] = J.rigid_from_x(x[c]) @ T[c]
    out.H = np.array(T)
    out.N = Nbig
    s0sq = ss / (m - 6 * F) if m > 6 * F else float("nan")
    out.s0 = float(np.sqrt(s0sq))
    Ninv = np.linalg.inv(Nbig)
    H = out.H
    cov = np.zeros((n_clouds, 6, 6))
    cov[~used] = np.nan
    Jc = {c: lever(np.eye(3), H[c][:3, 3]) for c in slot}
    for c, k in slot.items():
        cov[c] = s0sq * Jc[c] @ Ninv[6 * k:6 * k + 6, 6 * k:6 * k + 6] @ Jc[c].T
    edge_cov = np.zeros((len(edges), 6, 6))
    for e, (a, b) in enumerate(edges):
        Rt = H[a][:3, :3].T
        Ga = lever(Rt, H[b][:3, 3] - H[a][:3, 3])
        Gb = lever(Rt, np.zeros(3))
        C = Gb @ cov[b] @ Gb.T + Ga @ cov[a] @ Ga.T
        if a in slot and b in slot:
            i, j = 6 * slot[a], 6 * slot[b]
            M = Ga @ (s0sq * Jc[a] @ Ninv[i:i + 6, j:j + 6] @ Jc[b].T) @ Gb.T
            C -= M + M.T
        edge_cov[e] = C
    if not np.isfinite(s0sq):
        cov[:] = np.nan
        edge_cov[:] = np.nan
    out.cov, out.edge_cov = cov, edge_cov
    return out
