"""The a-posteriori covariances of a joint registration with relative pose observations (DESIGN.md
§6.13) restated in NumPy, for the tests; joint_prior_cov_rule.py states them with pose priors.

As there, the final iteration of a finished restatement run `res` is repeated from the poses the
same call stopped one iteration earlier gives, with the selection and normals of `res`: the edges'
kept rows, the priors' and the observations' blocks at those poses, the joint matrix N with them
and its solution x.  Then s0^2 = (sum_e r_e^T r_e + sum_c v_c^T W_c v_c + sum_k v_k^T W_k v_k) /
(sum_e n_e + sum_c m_c + sum_k m_k - 6 F) with v_k = B_b x_b - B_a x_a - l_k and m_k the non-zero
weights of each read observation, and C_c = s0^2 J_c' (N^-1)_cc J_c'^T as without them."""
import numpy as np

from oracle import joint_oracle as J
import joint_relative_oracle as JRO
from joint_cov_rule import FinalIteration, lever


def final_iteration(clouds, edges, res, fixed=(0,), H0=None, prior_poses=None, prior_weights=None,
                    relative_pairs=None, relative_poses=None, relative_weights=None, min_planarity: float = 0.3,
                    **kw) -> FinalIteration:
    """The final iteration of `res` = JRO.simpleicp_joint(clouds, edges, fixed=fixed, H0=H0, ...,
    min_planarity=min_planarity, **kw), and its covariances."""
    edges = np.asarray(edges, dtype=np.int64)
    n_clouds = len(clouds)
    nrm = {e: (res.normals[e], res.planarity[e]) for e in range(len(edges))}
    kw = {k: v for k, v in kw.items() if k not in ("max_iterations", "normals")}
    obs = dict(prior_poses=prior_poses, prior_weights=prior_weights, relative_pairs=relative_pairs,
               relative_poses=relative_poses, relative_weights=relative_weights)
    pre = JRO.simpleicp_joint(clouds, edges, fixed=fixed, H0=H0, min_planarity=min_planarity,
                              max_iterations=len(res.log) - 1, normals=nrm, **obs, **kw)
    T = [np.array(h) for h in pre.H]
    used = np.zeros(n_clouds, dtype=bool)
    used[edges.ravel()] = True
    is_fixed = np.zeros(n_clouds, dtype=bool)
    is_fixed[list(fixed)] = True
    slot = {c: k for k, c in enumerate(c for c in range(n_clouds) if used[c] and not is_fixed[c])}
    F = len(slot)
    P1 = {e: np.asarray(clouds[a], dtype=np.float64)[res.idx_fix[e]] for e, (a, _) in enumerate(edges)}
    nv = {e: np.asarray(res.normals[e], dtype=np.float64) for e in range(len(edges))}
    rows, _ = J._edge_rows(clouds, edges, T, P1, nv, res.planarity, {}, min_planarity)
    priors = JRO.JPO.prior_terms(T, slot, prior_poses, prior_weights)
    rels = JRO.relative_terms(T, slot, relative_pairs, relative_poses, relative_weights)
    Nbig, gbig = JRO.dense_matrix(edges, rows, slot, F, priors, rels)
    xs = np.linalg.solve(Nbig, gbig)
    x = {c: xs[6 * k:6 * k + 6] for c, k in slot.items()}
    out = FinalIteration(slot=slot)
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
    for p in priors:
        v = p.J @ xs[6 * p.slot:6 * p.slot + 6] - p.l
        ss += float(v @ (p.w * v))
        m += int(np.count_nonzero(p.w))
    for r in rels:
        u = np.zeros(6)
        if r.sb is not None:
            u += r.Bb @ xs[6 * r.sb:6 * r.sb + 6]
        if r.sa is not None:
            u -= r.Ba @ xs[6 * r.sa:6 * r.sa + 6]
        v = u - r.l
        ss += float(v @ (r.w * v))
        m += int(np.count_nonzero(r.w))
    for c in slot:
        T[c] = J.rigid_from_x(x[c]) @ T[c]
    out.H = np.array(T)
    out.N = Nbig
    out.priors = priors
    out.rels = rels  # the observation terms of the final iteration (JRO.RelTerm)
    s0sq = ss / (m - 6 * F) if m > 6 * F else float("nan")
    out.s0 = float(np.sqrt(s0sq))
    Ninv = np.linalg.inv(Nbig)
    cov = np.zeros((n_clouds, 6, 6))
    cov[~used] = np.nan
    for c, k in slot.items():
        Jc = lever(np.eye(3), out.H[c][:3, 3])
        cov[c] = s0sq * Jc @ Ninv[6 * k:6 * k + 6, 6 * k:6 * k + 6] @ Jc.T
    if not np.isfinite(s0sq):
        cov[:] = np.nan
    out.cov = cov
    return out
