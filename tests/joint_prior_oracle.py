"""The joint registration with pose priors (DESIGN.md §6.12) restated in NumPy/SciPy for the tests,
on top of the restatement without priors (oracle/joint_oracle.py), whose selection, match,
rejection, rows, pose update and stop rule it uses unchanged.

A free cloud c with an observed pose P_c and weights w_c, not all 0, adds
(J_c x_c - l_c)^T diag(w_c) (J_c x_c - l_c) to the minimisation, with l_c = (rotvec(R_P R_c^T),
o_P - o_c) at the current pose and J_c = [[I, 0], [-[o_c]x, I]] (x_c about the world origin, as in
the oracle).  The terms are summed after the edges' terms, in free-cloud order, by both solvers.
Without a prior that is read, simpleicp_joint here returns what J.simpleicp_joint returns, bit for
bit (test_joint_prior_host.py checks it)."""
from dataclasses import dataclass
from typing import List

import numpy as np
from scipy import sparse
from scipy.sparse import linalg as sparse_linalg
from scipy.spatial.transform import Rotation

from oracle import joint_oracle as J
from oracle.linearized_oracle import change, sample_std


@dataclass
class PriorTerm:
    slot: int           # the cloud's free slot
    N: np.ndarray       # J^T W J
    g: np.ndarray       # J^T W l
    l: np.ndarray       # the observation (rotvec(R_P R_c^T), o_P - o_c)
    J: np.ndarray       # [[I, 0], [-[o_c]x, I]]
    w: np.ndarray


def prior_terms(T, slot, prior_poses, prior_weights) -> List[PriorTerm]:
    """The pose priors read at the poses T, in free-cloud order: those of free clouds with a
    non-zero weight."""
    out = []
    if prior_weights is None:
        return out
    for c, k in slot.items():
        w = np.asarray(prior_weights[c], dtype=np.float64)
        if not np.any(w != 0.0):
            continue
        P = np.asarray(prior_poses[c], dtype=np.float64)
        l = np.concatenate((Rotation.from_matrix(P[:3, :3] @ T[c][:3, :3].T).as_rotvec(), P[:3, 3] - T[c][:3, 3]))
        Jc = np.eye(6)
        Jc[3:, :3] = -J.skew(T[c][:3, 3])
        out.append(PriorTerm(k, Jc.T @ (w[:, None] * Jc), Jc.T @ (w * l), l, Jc, w))
    return out


def joint_terms(edges, rows, slot, priors=()):
    """J._joint_blocks' terms of the edges, then per pose prior ("N", i, i, J^T W J) and
    ("g", i, J^T W l), i = 6 x the cloud's free slot."""
    yield from J._joint_blocks(edges, rows, slot)
    for p in priors:
        yield "N", 6 * p.slot, 6 * p.slot, p.N
        yield "g", 6 * p.slot, p.g


def dense_matrix(edges, rows, slot, F, priors=()):
    """The joint normal matrix and right-hand side, summed as J._dense_solve sums them."""
    Nbig = np.zeros((6 * F, 6 * F))
    gbig = np.zeros(6 * F)
    for t in joint_terms(edges, rows, slot, priors):
        if t[0] == "N":
            Nbig[t[1]:t[1] + 6, t[2]:t[2] + 6] += t[3]
        else:
            gbig[t[1]:t[1] + 6] += t[2]
    return Nbig, gbig


def _solve(edges, rows, slot, F, priors, solver):
    """J._dense_solve or J._sparse_solve of the system with the priors' terms."""
    if solver == "dense":
        Nbig, gbig = dense_matrix(edges, rows, slot, F, priors)
        np.linalg.cholesky(Nbig)
        return np.linalg.solve(Nbig, gbig)
    ii, jj, vv = [], [], []
    gbig = np.zeros(6 * F)
    r6 = np.repeat(np.arange(6), 6)
    c6 = np.tile(np.arange(6), 6)
    for t in joint_terms(edges, rows, slot, priors):
        if t[0] == "N":
            ii.append(t[1] + r6)
            jj.append(t[2] + c6)
            vv.append(t[3].ravel())
        else:
            gbig[t[1]:t[1] + 6] += t[2]
    Nbig = sparse.csc_matrix((np.concatenate(vv), (np.concatenate(ii), np.concatenate(jj))), shape=(6 * F, 6 * F))
    return sparse_linalg.spsolve(Nbig, gbig)


def simpleicp_joint(clouds, edges, fixed=(0,), H0=None, correspondences: int = 1000, neighbors: int = 10,
                    min_planarity: float = 0.3, max_overlap_distance: float = np.inf, min_change: float = 1.0,
                    max_iterations: int = 100, normals: J.Normals = None, solver: str = "dense", prior_poses=None,
                    prior_weights=None) -> J.JointResult:
    """J.simpleicp_joint with the pose priors ``prior_poses`` (n_clouds, 4, 4) and ``prior_weights``
    (n_clouds, 6) added to every iteration's system; the other arguments and the result as there."""
    if solver not in ("dense", "sparse"):
        raise ValueError("solver must be 'dense' or 'sparse'")
    edges, T, free = J._start(clouds, edges, fixed, H0)
    slot = {c: k for k, c in enumerate(free)}
    F = len(free)
    res = J.JointResult()
    P1, nrm, pl = J._setup_edges(clouds, edges, T, res, correspondences, neighbors, max_overlap_distance, normals)
    trees = {}
    prev = {}
    for it in range(max_iterations):
        rows, log = J._edge_rows(clouds, edges, T, P1, nrm, pl, trees, min_planarity)
        priors = prior_terms(T, slot, prior_poses, prior_weights)
        xs = _solve(edges, rows, slot, F, priors, solver)
        x = {c: xs[6 * k:6 * k + 6] for c, k in slot.items()}
        conv = it > 0
        for e, (a, b) in enumerate(edges):
            A, l, Ad = rows[e]
            if A.shape[0] < 6:
                continue
            xi = Ad @ (x.get(b, np.zeros(6)) - x.get(a, np.zeros(6)))
            r = A @ xi - l
            log[e].mean, log[e].std, log[e].xi = float(r.mean()), sample_std(r), xi
            if e in prev:
                m0, s0 = prev[e]
                conv = conv and change(log[e].mean, m0) < min_change and change(log[e].std, s0) < min_change
            else:
                conv = False
            prev[e] = (log[e].mean, log[e].std)
        for c in free:
            T[c] = J.rigid_from_x(x[c]) @ T[c]
        res.log.append(log)
        if conv:
            res.converged = True
            break
    res.H = np.array(T)
    res.R = [np.linalg.inv(T[a]) @ T[b] for a, b in edges]
    return res
