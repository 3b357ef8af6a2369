"""The joint registration with relative pose observations (DESIGN.md §6.13) restated in NumPy/SciPy
for the tests, on top of the restatement with pose priors (joint_prior_oracle.py), whose edges,
priors, pose update and stop rule it uses unchanged.

Observation k of clouds (a, b), with an observed Z of T_a^-1 T_b and weights w, not all 0, and a
free end, adds (u_k - l_k)^T diag(w) (u_k - l_k) to the minimisation, with
l_k = (rotvec(R_Z R_ab^T), t_Z - t_ab), R_ab = R_a^T R_b, t_ab = R_a^T (o_b - o_a) at the current
poses and u_k = G_b J_b x_b - G_a J_a x_a, G_b = diag(R_a^T, R_a^T),
G_a = [[R_a^T, 0], [-R_a^T [o_b - o_a]x, R_a^T]], J_c = [[I, 0], [-[o_c]x, I]] (x_c about the world
origin, as in the oracle); a fixed end has no unknowns.  The terms are summed after the edges' and
the priors', in ascending k, by both solvers.  Without an observation that is read,
simpleicp_joint here returns what JPO.simpleicp_joint returns, bit for bit
(test_joint_relative_host.py checks it)."""
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
from scipy import sparse
from scipy.sparse import linalg as sparse_linalg
from scipy.spatial.transform import Rotation

from oracle import joint_oracle as J
from oracle.linearized_oracle import change, sample_std
import joint_prior_oracle as JPO


@dataclass
class RelTerm:
    sa: Optional[int]   # the free slots of clouds a and b (None: fixed)
    sb: Optional[int]
    Ba: np.ndarray      # G_a J_a
    Bb: np.ndarray      # G_b J_b
    l: np.ndarray       # the observation (rotvec(R_Z R_ab^T), t_Z - t_ab)
    w: np.ndarray


def observe(Ta, Tb, Z) -> np.ndarray:
    """l = (rotvec(R_Z R_ab^T), t_Z - t_ab) of the observed Z of T_a^-1 T_b at the poses Ta, Tb."""
    Ra = Ta[:3, :3]
    Rab = Ra.T @ Tb[:3, :3]
    tab = Ra.T @ (Tb[:3, 3] - Ta[:3, 3])
    return np.concatenate((Rotation.from_matrix(Z[:3, :3] @ Rab.T).as_rotvec(), Z[:3, 3] - tab))


def jacobians(Ta, Tb):
    """(G_a J_a, G_b J_b): u = G_b J_b x_b - G_a J_a x_a with x_c about the world origin."""
    Ra = Ta[:3, :3]
    Ga = np.zeros((6, 6))
    Ga[:3, :3] = Ga[3:, 3:] = Ra.T
    Ga[3:, :3] = -Ra.T @ J.skew(Tb[:3, 3] - Ta[:3, 3])
    Gb = np.zeros((6, 6))
    Gb[:3, :3] = Gb[3:, 3:] = Ra.T
    out = []
    for G, T in ((Ga, Ta), (Gb, Tb)):
        Jc = np.eye(6)
        Jc[3:, :3] = -J.skew(T[:3, 3])
        out.append(G @ Jc)
    return out


def relative_terms(T, slot, pairs, poses, weights) -> List[RelTerm]:
    """The relative observations read at the poses T, in ascending order: those with a non-zero
    weight and a free end."""
    out = []
    if pairs is None:
        return out
    poses, weights = np.asarray(poses, dtype=np.float64), np.asarray(weights, dtype=np.float64)
    for (a, b), Z, w in zip(np.asarray(pairs), poses, weights):
        a, b = int(a), int(b)
        if not np.any(w != 0.0) or (a not in slot and b not in slot):
            continue
        Ba, Bb = jacobians(T[a], T[b])
        out.append(RelTerm(slot.get(a), slot.get(b), Ba, Bb, observe(T[a], T[b], Z), w))
    return out


def joint_terms(edges, rows, slot, priors=(), rels=()):
    """JPO.joint_terms (the edges, then the priors), then per relative observation, for each free
    end c (a, then b) ("N", i_c, i_c, B_c^T W B_c) and ("g", i_c, -+B_c^T W l), then for two free
    ends ("N", i_a, i_b, -B_a^T W B_b) and ("N", i_b, i_a, -B_b^T W B_a)."""
    yield from JPO.joint_terms(edges, rows, slot, priors)
    for r in rels:
        for s, B, sg in ((r.sa, r.Ba, -1.0), (r.sb, r.Bb, 1.0)):
            if s is not None:
                yield "N", 6 * s, 6 * s, B.T @ (r.w[:, None] * B)
                yield "g", 6 * s, sg * (B.T @ (r.w * r.l))
        if r.sa is not None and r.sb is not None:
            yield "N", 6 * r.sa, 6 * r.sb, -(r.Ba.T @ (r.w[:, None] * r.Bb))
            yield "N", 6 * r.sb, 6 * r.sa, -(r.Bb.T @ (r.w[:, None] * r.Ba))


def dense_matrix(edges, rows, slot, F, priors=(), rels=()):
    """The joint normal matrix and right-hand side, summed as JPO.dense_matrix sums them."""
    Nbig = np.zeros((6 * F, 6 * F))
    gbig = np.zeros(6 * F)
    for t in joint_terms(edges, rows, slot, priors, rels):
        if t[0] == "N":
            Nbig[t[1]:t[1] + 6, t[2]:t[2] + 6] += t[3]
        else:
            gbig[t[1]:t[1] + 6] += t[2]
    return Nbig, gbig


def _solve(edges, rows, slot, F, priors, rels, solver):
    """JPO._solve with the observations' terms."""
    if solver == "dense":
        Nbig, gbig = dense_matrix(edges, rows, slot, F, priors, rels)
        np.linalg.cholesky(Nbig)
        return np.linalg.solve(Nbig, gbig)
    ii, jj, vv = [], [], []
    gbig = np.zeros(6 * F)
    r6 = np.repeat(np.arange(6), 6)
    c6 = np.tile(np.arange(6), 6)
    for t in joint_terms(edges, rows, slot, priors, rels):
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
                    prior_weights=None, relative_pairs=None, relative_poses=None,
                    relative_weights=None) -> J.JointResult:
    """JPO.simpleicp_joint with the relative observations ``relative_pairs`` (n_rel, 2),
    ``relative_poses`` (n_rel, 4, 4) and ``relative_weights`` (n_rel, 6) added to every iteration's
    system; the other arguments and the result as there."""
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
        priors = JPO.prior_terms(T, slot, prior_poses, prior_weights)
        rels = relative_terms(T, slot, relative_pairs, relative_poses, relative_weights)
        xs = _solve(edges, rows, slot, F, priors, rels, solver)
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
