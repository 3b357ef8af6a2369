"""NumPy/SciPy restatement of the joint (multi-scan) linearised registration of
sicp_register_joint / simpleicp_joint (DESIGN.md §6.9).

Each cloud c has a pose T_c (world <- cloud) starting at H0[c]; the clouds in `fixed` keep theirs.
Edge e = (a, b) is registered like the pair (a, b) of the linearised variant
(linearized_oracle.simpleicp_linearized) from R_e = T_a^-1 T_b: selection, overlap filter and
normals once under the initial R_e, then per iteration the match of cloud b moved by R_e, the
median / MAD rejection and the rows A_e x = l_e in frame a.  The increments are solved jointly:
one x_c = (alpha, t) per free cloud in the world frame about the origin, the edge's increment
xi_e = Ad(T_a^-1) (x_b - x_a), minimising sum_e |A_e xi_e - l_e|^2 over the edges with >= 6 kept
rows (np.linalg.solve of the dense normal equations, or scipy.sparse.linalg.spsolve of the same
system assembled sparsely under solver="sparse"); then T_c <- dH(x_c) T_c with the rigid Euler dH of
the pair path.  Converged at iteration i > 0 when every edge that took part meets the linearised
stop rule.  first_iteration_sums returns the per-edge sums of one iteration, from which a test
can assemble the joint system in any variables it likes."""
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Union

import numpy as np
from scipy import sparse, spatial
from scipy.sparse import linalg as sparse_linalg

from .linearized_oracle import (change, estimate_normals, euler_angles_to_rotation_matrix, median_upper,
                                mad_upper, sample_std, select_in_range, select_n_points)


def skew(v: np.ndarray) -> np.ndarray:
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def ad_world_to_frame(T_a: np.ndarray) -> np.ndarray:
    """The 6 x 6 map carrying a world-frame small motion y -> y + w x y + t into the frame of T_a:
    (R^T w, R^T (t - p x w)) with R, p the rotation and translation of T_a."""
    R, p = T_a[:3, :3], T_a[:3, 3]
    Ad = np.zeros((6, 6))
    Ad[:3, :3] = R.T
    Ad[3:, 3:] = R.T
    Ad[3:, :3] = -R.T @ skew(p)
    return Ad


def rigid_from_x(x: np.ndarray) -> np.ndarray:
    H = np.eye(4)
    H[:3, :3] = euler_angles_to_rotation_matrix(x[0], x[1], x[2])
    H[:3, 3] = x[3:6]
    return H


@dataclass
class EdgeIteration:
    n_kept: int = 0
    mean: float = float("nan")
    std: float = float("nan")
    xi: Optional[np.ndarray] = None
    keep: Optional[np.ndarray] = None


@dataclass
class JointResult:
    H: np.ndarray = None                        # (n_clouds, 4, 4) final poses
    R: List[np.ndarray] = field(default_factory=list)   # per edge: final T_a^-1 T_b
    log: List[List[EdgeIteration]] = field(default_factory=list)  # per iteration, per edge
    converged: bool = False
    idx_fix: Dict[int, np.ndarray] = field(default_factory=dict)
    normals: Dict[int, np.ndarray] = field(default_factory=dict)
    planarity: Dict[int, np.ndarray] = field(default_factory=dict)


def _workers(n_queries: int) -> int:
    """Threads for an exact k-d tree query of n_queries points: one below 100 000, where starting
    threads costs more than the query (thousands of edges of a few thousand points each); all
    cores above.  The neighbours do not depend on it."""
    return 1 if n_queries < 100_000 else -1


Normals = Union[Dict[int, tuple], Callable[[int, np.ndarray], tuple], None]


def _setup_edges(clouds, edges, T, res, correspondences, neighbors, max_overlap_distance, normals: Normals):
    """Per edge, once: selection, overlap filter and normals under the initial R_e.  Returns the
    selected fixed points, their normals and planarity, per edge."""
    P1, nrm, pl = {}, {}, {}
    for e, (a, b) in enumerate(edges):
        Xf = np.asarray(clouds[a], dtype=np.float64)
        R = np.linalg.inv(T[a]) @ T[b]
        idx = np.arange(Xf.shape[0])
        if np.isfinite(max_overlap_distance) and max_overlap_distance > 0:
            Xm = np.asarray(clouds[b], dtype=np.float64) @ R[:3, :3].T + R[:3, 3]
            idx = select_in_range(Xf, Xm, max_overlap_distance, workers=_workers(Xf.shape[0]))
        idx = select_n_points(idx, correspondences)
        if callable(normals):
            nv, pv = normals(e, idx)
        elif normals is not None and e in normals:
            nv, pv = normals[e]
        else:
            nv, pv = estimate_normals(Xf, idx, neighbors)
        P1[e], nrm[e], pl[e] = Xf[idx], np.asarray(nv, dtype=np.float64), np.asarray(pv, dtype=np.float64)
        res.idx_fix[e], res.normals[e], res.planarity[e] = idx, nrm[e], pl[e]
    return P1, nrm, pl


def _edge_rows(clouds, edges, T, P1, nrm, pl, trees, min_planarity):
    """One iteration's match and rejection of every edge: per edge the kept rows (A, l) in frame a
    with Ad(T_a^-1), and the log entry."""
    rows = []
    log = []
    for e, (a, b) in enumerate(edges):
        if P1[e].shape[0] == 0:  # no overlap: no rows, the edge takes no part
            rows.append((np.empty((0, 6)), np.empty(0), ad_world_to_frame(T[a])))
            log.append(EdgeIteration(0, keep=np.zeros(0, dtype=bool)))
            continue
        R = np.linalg.inv(T[a]) @ T[b]
        if b not in trees:
            trees[b] = spatial.cKDTree(np.asarray(clouds[b], dtype=np.float64))
        Xb = np.asarray(clouds[b], dtype=np.float64)
        # nearest neighbour of R^-1 p1 in cloud b, i.e. of p1 in cloud b moved by R
        Ri = np.linalg.inv(R)
        _, nn = trees[b].query(P1[e] @ Ri[:3, :3].T + Ri[:3, 3], k=1, workers=_workers(P1[e].shape[0]))
        P2 = Xb[nn] @ R[:3, :3].T + R[:3, 3]
        n = nrm[e]
        d = np.einsum("ij,ij->i", P2 - P1[e], n)
        med = median_upper(d)
        sig = 1.4826 * mad_upper(d)
        keep = ~((np.abs(d - med) > 3.0 * sig) | (pl[e] < min_planarity))
        p1, p2, nk = P1[e][keep], P2[keep], n[keep]
        A = np.empty((p1.shape[0], 6))
        A[:, 0] = -p2[:, 2] * nk[:, 1] + p2[:, 1] * nk[:, 2]
        A[:, 1] = p2[:, 2] * nk[:, 0] - p2[:, 0] * nk[:, 2]
        A[:, 2] = -p2[:, 1] * nk[:, 0] + p2[:, 0] * nk[:, 1]
        A[:, 3:6] = nk
        l = np.einsum("ij,ij->i", nk, p1 - p2)
        rows.append((A, l, ad_world_to_frame(T[a])))
        log.append(EdgeIteration(int(keep.sum()), keep=keep))
    return rows, log


def _start(clouds, edges, fixed, H0):
    edges = np.asarray(edges, dtype=np.int64)
    n_clouds = len(clouds)
    T = [np.eye(4) if H0 is None else np.array(H0[c], dtype=np.float64) for c in range(n_clouds)]
    used = np.zeros(n_clouds, dtype=bool)
    used[edges.ravel()] = True
    is_fixed = np.zeros(n_clouds, dtype=bool)
    is_fixed[list(fixed)] = True
    free = [c for c in range(n_clouds) if used[c] and not is_fixed[c]]
    return edges, T, free


def _joint_blocks(edges, rows, slot):
    """The joint normal equations over the free clouds as the terms both solvers sum, in the order
    they sum them: per edge with >= 6 kept rows, N = Ad^T A^T A Ad and g = Ad^T A^T l; for each
    free end c (a, then b) ("N", i, i, N) and ("g", i, -g for a, +g for b), then for two free ends
    ("N", i_a, i_b, -N) and ("N", i_b, i_a, -N); i = 6 x the cloud's free slot."""
    for e, (a, b) in enumerate(edges):
        A, l, Ad = rows[e]
        if A.shape[0] < 6:
            continue
        N = Ad.T @ (A.T @ A) @ Ad
        g = Ad.T @ (A.T @ l)
        for c, s in ((a, -1.0), (b, 1.0)):
            if c in slot:
                i = 6 * slot[c]
                yield "N", i, i, N
                yield "g", i, s * g
        if a in slot and b in slot:
            i, j = 6 * slot[a], 6 * slot[b]
            yield "N", i, j, -N
            yield "N", j, i, -N


def _dense_solve(edges, rows, slot, F):
    """np.linalg.solve of the dense normal equations, after a Cholesky check of definiteness
    (LinAlgError: not positive definite)."""
    Nbig = np.zeros((6 * F, 6 * F))
    gbig = np.zeros(6 * F)
    for t in _joint_blocks(edges, rows, slot):
        if t[0] == "N":
            Nbig[t[1]:t[1] + 6, t[2]:t[2] + 6] += t[3]
        else:
            gbig[t[1]:t[1] + 6] += t[2]
    np.linalg.cholesky(Nbig)
    return np.linalg.solve(Nbig, gbig)


def _sparse_solve(edges, rows, slot, F):
    """The same terms assembled as a scipy.sparse matrix and solved by spsolve (no definiteness
    check)."""
    ii, jj, vv = [], [], []
    gbig = np.zeros(6 * F)
    r6 = np.repeat(np.arange(6), 6)
    c6 = np.tile(np.arange(6), 6)
    for t in _joint_blocks(edges, rows, slot):
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
                    max_iterations: int = 100, normals: Normals = None, solver: str = "dense") -> JointResult:
    """``normals`` maps an edge number to (normals, planarity) of its selected fixed points, or is a
    function (edge, selected indices) -> (normals, planarity); either then replaces the estimate
    (lock-step comparisons hand over the device's float32 normals).  ``solver`` "dense" solves the
    joint normal equations with np.linalg.solve after a Cholesky check of definiteness, "sparse"
    with scipy.sparse.linalg.spsolve (for more free clouds than a dense matrix holds)."""
    if solver not in ("dense", "sparse"):
        raise ValueError("solver must be 'dense' or 'sparse'")
    edges, T, free = _start(clouds, edges, fixed, H0)
    slot = {c: k for k, c in enumerate(free)}
    F = len(free)
    res = JointResult()

    # ---- per edge, once: selection, overlap filter and normals under the initial R_e
    P1, nrm, pl = _setup_edges(clouds, edges, T, res, correspondences, neighbors, max_overlap_distance, normals)
    trees = {}

    prev = {}
    for it in range(max_iterations):
        rows, log = _edge_rows(clouds, edges, T, P1, nrm, pl, trees, min_planarity)
        # ---- joint normal equations over the free clouds
        xs = (_sparse_solve if solver == "sparse" else _dense_solve)(edges, rows, slot, F)
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
            T[c] = rigid_from_x(x[c]) @ T[c]
        res.log.append(log)
        if conv:
            res.converged = True
            break
    res.H = np.array(T)
    res.R = [np.linalg.inv(T[a]) @ T[b] for a, b in edges]
    return res


@dataclass
class EdgeSums:
    N: np.ndarray       # (n_edges, 6, 6) A^T A of the kept rows, frame a, about frame a's origin
    g: np.ndarray       # (n_edges, 6) A^T l
    n_kept: np.ndarray  # (n_edges,)
    T_a: np.ndarray     # (n_edges, 4, 4) the start pose of each edge's cloud a
    free: List[int] = field(default_factory=list)  # the free clouds in free-cloud order


def first_iteration_sums(clouds, edges, fixed=(0,), H0=None, correspondences: int = 1000, neighbors: int = 10,
                         min_planarity: float = 0.3, max_overlap_distance: float = np.inf,
                         normals: Normals = None) -> EdgeSums:
    """The first iteration of simpleicp_joint up to its solve: per edge the sums of the kept rows
    A_e x = l_e in frame a (A^T A, A^T l, the count) and T_a, the same rows the joint system of that
    iteration is built from, without building or solving it."""
    edges, T, free = _start(clouds, edges, fixed, H0)
    P1, nrm, pl = _setup_edges(clouds, edges, T, JointResult(), correspondences, neighbors, max_overlap_distance,
                               normals)
    rows, log = _edge_rows(clouds, edges, T, P1, nrm, pl, {}, min_planarity)
    return EdgeSums(N=np.array([A.T @ A for A, _, _ in rows]).reshape(-1, 6, 6),
                    g=np.array([A.T @ l for A, l, _ in rows]).reshape(-1, 6),
                    n_kept=np.array([lg.n_kept for lg in log], dtype=np.int64),
                    T_a=np.array([T[a] for a, _ in edges]).reshape(-1, 4, 4), free=free)
