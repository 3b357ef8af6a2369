"""sicp_get_joint_selected_covariances / simpleicp_joint(covariances="selected") on the GPU
(DESIGN.md §6.14): after a dense call the bits of sicp_get_joint_covariances; after a sparse call
the selected inversion of the sparse factor, in lock-step with the NumPy rules (joint_cov_rule.py,
joint_prior_cov_rule.py, joint_relative_cov_rule.py) and against the dense request on the same
problem; past the dense cap against J' N'^-1 J'^T from sparse solves of N' assembled exactly from
the oracle's first-iteration sums; the structure (fixed, unused, symmetric), parked edges outside
the pattern, separate components, georeferenced coordinates, the call order and the end-to-end call.

Tolerances follow test_gpu_joint_cov: s0 to 1e-12 relative, every sigma to SIG = 10 kappa u and
every correlation to CORR = 100 kappa u absolute, kappa the condition number of the rule's N (past
the dense cap, of N' from its extreme eigenvalues by scipy's eigsh)."""
import numpy as np
import pytest

import simpleicp_b200 as sb
from oracle import joint_oracle as J
from simpleicp_b200 import _capi
from simpleicp_b200._capi import SicpError

import joint_cov_rule as JC
import joint_prior_cov_rule as JP
import joint_relative_cov_rule as JRC
from test_gpu_joint import _lockstep as _lockstep_edges, _pair, _params, strip
from test_gpu_joint_cov import _corr, _lever, _one_pair_state, _sig
from test_gpu_joint_graphs import _block, _oracle_sums, _skew
from test_gpu_joint_priors import _lockstep as _lockstep_priors, _noisy, _ring_priors
from test_gpu_joint_relative import _joint, _lockstep as _lockstep_rel, _ring_rel, _strip127_rel
from test_joint_host import ring

pytestmark = pytest.mark.gpu

S0_TOL = 1e-12


@pytest.fixture(scope="module")
def eng():
    e = _capi.Engine(0)
    yield e
    e.close()


def _tols(N):
    ku = np.linalg.cond(N) * np.finfo(np.float64).eps / 2
    return max(10 * ku, 1e-12), max(100 * ku, 1e-12), ku


def _agree(label, cov, ecov, s0, rcov, recov, rs0, free, sig_tol, corr_tol):
    """cov / ecov / s0 against a reference over the free clouds and the edges (recov None: clouds
    only); both blocks exactly symmetric."""
    assert abs(s0 - rs0) <= S0_TOL * rs0, (label, s0, rs0)
    d_sig = np.abs(_sig(cov[free]) / _sig(rcov[free]) - 1).max()
    d_corr = np.abs(_corr(cov[free]) - _corr(rcov[free])).max()
    if recov is not None:
        d_sig = max(d_sig, np.abs(_sig(ecov) / _sig(recov) - 1).max())
        d_corr = max(d_corr, np.abs(_corr(ecov) - _corr(recov)).max())
    print(f"{label}: s0 rel {abs(s0 / rs0 - 1):.2e}, sigma rel {d_sig:.2e} (tol {sig_tol:.1e}), "
          f"correlation abs {d_corr:.2e} (tol {corr_tol:.1e})")
    assert d_sig < sig_tol and d_corr < corr_tol, (label, d_sig, sig_tol, d_corr, corr_tol)
    assert np.array_equal(cov, np.swapaxes(cov, 1, 2), equal_nan=True)
    assert np.array_equal(ecov, np.swapaxes(ecov, 1, 2), equal_nan=True)


def _sel(eng, n_c, n_e):
    return eng.joint_selected_covariances(n_c, n_e)


def _same_bits(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a[:2], b[:2])) and np.float64(a[2]).tobytes() == \
        np.float64(b[2]).tobytes()


def _dense_request(eng, scans, edges, fixed, H0, P=None, W=None, rel=(), its=30):
    _joint(eng, 0, scans, edges, fixed, H0, P, W, rel=rel, max_iterations=its)
    return eng.joint_covariances(len(scans), len(edges))


# --------------------------------------------------------------------------- after a dense call
def test_after_a_dense_call_the_bits_of_sicp_get_joint_covariances(eng):
    scans, truth, H0, edges = ring()
    P, W = _ring_priors(truth)
    rel = _ring_rel(truth)
    n_c, n_e = len(scans), len(edges)
    _joint(eng, 0, scans, edges, (0,), H0, P, W, rel=rel)
    old = eng.joint_covariances(n_c, n_e)
    new = _sel(eng, n_c, n_e)
    assert _same_bits(old, new)
    _joint(eng, 0, scans, edges, (0,), H0, P, W, rel=rel)
    new2 = _sel(eng, n_c, n_e)  # asked first this time
    old2 = eng.joint_covariances(n_c, n_e)
    assert _same_bits(new2, old2) and _same_bits(old, new2)
    # the old entry point keeps refusing after a sparse call, also after the new request
    _joint(eng, 1, scans, edges, (0,), H0, P, W, rel=rel)
    for _ in range(2):
        with pytest.raises(SicpError, match="covariances need joint_solver 0") as ei:
            eng.joint_covariances(n_c, n_e)
        assert ei.value.code == _capi.SICP_ERR_STATE
        _sel(eng, n_c, n_e)


# --------------------------------------------------------------------------- against the rules
@pytest.mark.parametrize("problem", ["ring", "strip127", "strip255"])
def test_sparse_lockstep_against_the_rule(eng, problem):
    if problem == "ring":
        scans, truth, H0, edges = ring()
        its = 30
    elif problem == "strip127":
        scans, truth, H0, edges = strip(128, 50_000, 400)
        its = 20
    else:
        scans, truth, H0, edges = strip(256, 20_000, 800)
        its = 4
    eng.set_option("joint_solver", 1)
    try:
        H, out, logs, run = _lockstep_edges(eng, scans, H0, edges, (0,), max_iterations=its)
    finally:
        eng.set_option("joint_solver", 0)
    assert np.abs(H - run.H).max() < 1e-9
    ref = JC.final_iteration(scans, edges, run, H0=H0, max_overlap_distance=1.0)
    cov, ecov, s0 = _sel(eng, len(scans), len(edges))
    sig_tol, corr_tol, _ = _tols(ref.N)
    free = np.arange(1, len(scans))
    _agree(f"sparse vs rule ({problem})", cov, ecov, s0, ref.cov, ref.edge_cov, ref.s0, free, sig_tol, corr_tol)
    assert np.array_equal(cov[0], np.zeros((6, 6)))
    d = _dense_request(eng, scans, edges, (0,), H0, its=its)
    _agree(f"sparse vs dense ({problem})", cov, ecov, s0, d[0], d[1], d[2], free, sig_tol, corr_tol)


@pytest.mark.parametrize("problem", ["ring_no_fixed", "strip127"])
def test_sparse_with_priors_against_the_rule(eng, problem):
    if problem == "ring_no_fixed":
        scans, truth, H0, edges = ring()
        P, W = _ring_priors(truth, anchor0=True)
        fixed, its = (), 30
    else:
        scans, truth, H0, edges = strip(128, 50_000, 400)
        P = _noisy(truth, 31, 0.03, 0.03)
        W = np.tile([0.01 ** 2 / np.deg2rad(0.03) ** 2] * 3 + [0.01 ** 2 / 0.03 ** 2] * 3, (128, 1))
        W[5:20, :3] = 0.0
        fixed, its = (0,), 20
    H, out, logs, ref, nrm = _lockstep_priors(eng, 1, scans, H0, edges, fixed, P, W, max_iterations=its)
    assert np.abs(H - ref.H).max() < 1e-9
    cov, ecov, s0 = _sel(eng, len(scans), len(edges))
    fi = JP.final_iteration(scans, edges, ref, fixed=fixed, H0=H0, prior_poses=P, prior_weights=W,
                            max_overlap_distance=1.0)
    free = list(fi.slot)
    sig_tol, corr_tol, _ = _tols(fi.N)
    _agree(f"sparse with priors vs rule ({problem})", cov, ecov, s0, fi.cov, None, fi.s0, free, sig_tol, corr_tol)
    d = _dense_request(eng, scans, edges, fixed, H0, P, W, its=its)
    _agree(f"sparse with priors vs dense ({problem})", cov, ecov, s0, d[0], d[1], d[2], free, sig_tol, corr_tol)


@pytest.mark.parametrize("problem", ["ring", "strip127"])
def test_sparse_with_relative_observations_against_the_rule(eng, problem):
    """strip127's observations (i, i + 13) join clouds no edge joins: blocks only they fill."""
    if problem == "ring":
        scans, truth, H0, edges = ring()
        rel, its = _ring_rel(truth), 30
    else:
        scans, truth, H0, edges = strip(128, 50_000, 400)
        rel, its = _strip127_rel(truth, edges), 20
        rel[2][5:20, :3] = 0.0
    H, out, logs, ref, nrm = _lockstep_rel(eng, 1, scans, H0, edges, (0,), rel, max_iterations=its)
    assert np.abs(H - ref.H).max() < 1e-9
    cov, ecov, s0 = _sel(eng, len(scans), len(edges))
    fi = JRC.final_iteration(scans, edges, ref, fixed=(0,), H0=H0, relative_pairs=rel[0], relative_poses=rel[1],
                             relative_weights=rel[2], max_overlap_distance=1.0)
    free = list(fi.slot)
    sig_tol, corr_tol, _ = _tols(fi.N)
    _agree(f"sparse with observations vs rule ({problem})", cov, ecov, s0, fi.cov, None, fi.s0, free, sig_tol,
           corr_tol)
    d = _dense_request(eng, scans, edges, (0,), H0, rel=rel, its=its)
    _agree(f"sparse with observations vs dense ({problem})", cov, ecov, s0, d[0], d[1], d[2], free, sig_tol,
           corr_tol)


def test_parked_pairs_in_one_component_from_the_forward_solves(eng):
    """The 127-cloud strip with three more edges between clouds 60 to 120 m apart: the filter parks
    them before the first iteration (no overlap), so they are not in the plan, and their cross
    blocks come from w_a^T w_b unless fill put the pair in the pattern.  Sparse against dense."""
    scans, truth, H0, edges = strip(128, 50_000, 400)
    E = np.vstack([edges, [(1, 100), (5, 60), (30, 120)]])
    res = []
    for solver in (0, 1):
        H, out = _joint(eng, solver, scans, E, (0,), H0, max_iterations=5)
        assert [o.status for o in out][-3:] == [_capi.SICP_ERR_NO_OVERLAP] * 3
        res.append(_sel(eng, len(scans), len(E)))
    (dc, de, ds), (cov, ecov, s0) = res
    sig_tol = corr_tol = 1e-6  # two solves of a strip's ill-conditioned system, in different unknowns
    _agree("parked pairs, sparse vs dense", cov, ecov, s0, dc, de, ds, np.arange(1, 128), sig_tol, corr_tol)


def _many_components(n_pieces=20):
    """n_pieces rings of 8 clouds side by side, 160 m apart, each with its own fixed cloud, and one
    edge between the first two rings' free clouds 1 and 9 without overlap: a parked pair of two
    components (their cross block is exactly 0), outside the pattern of a plan of more than one
    supernode."""
    scans, truth, H0, edges = ring()
    S, T, H, E, fixed = [], [], [], [], []
    for k in range(n_pieces):
        off = np.eye(4)
        off[0, 3] = 160.0 * k
        base = len(S)
        S += list(scans)
        T += [off @ t for t in truth]
        H += [off @ h for h in H0]
        E += [(base + a, base + b) for a, b in edges]
        fixed.append(base)
    E.append((1, 9))
    return S, np.array(T), np.array(H), np.array(E), tuple(fixed)


def test_separate_components_and_a_parked_pair_outside_the_pattern(eng):
    S, T, H0, E, fixed = _many_components()
    res = []
    for solver in (0, 1):
        H, out = _joint(eng, solver, S, E, fixed, H0)
        assert out[-1].status == _capi.SICP_ERR_NO_OVERLAP
        res.append(_sel(eng, len(S), len(E)))
    (dc, de, ds), (cov, ecov, s0) = res
    free = [c for c in range(len(S)) if c not in fixed]
    _agree("components, sparse vs dense", cov, ecov, s0, dc, de, ds, free, 1e-8, 1e-7)
    # the parked edge's C_e is G_b C_b G_b^T + G_a C_a G_a^T: the cross block is exactly 0
    Ha = H[1]
    d = H[9][:3, 3] - Ha[:3, 3]
    Ga, Gb = np.zeros((6, 6)), np.zeros((6, 6))
    Ga[:3, :3] = Ga[3:, 3:] = Gb[:3, :3] = Gb[3:, 3:] = Ha[:3, :3].T
    Ga[3:, :3] = -Ha[:3, :3].T @ _skew(d)
    want = Gb @ cov[9] @ Gb.T + Ga @ cov[1] @ Ga.T
    assert np.abs(ecov[-1] - want).max() <= 1e-12 * np.abs(want).max()


# --------------------------------------------------------------------------- past the dense cap
def _sparse_reference(sums, edges, H0, H, sample, P_w=None):
    """J' (N'^-1) J'^T for the sampled free clouds and the cross blocks of their edges, N' the first
    iteration's matrix in the sparse unknowns (levers p - o_c^0) plus diag(prior weights)."""
    from scipy import sparse
    from scipy.sparse.linalg import splu

    slot = {c: k for k, c in enumerate(sums.free)}
    F = len(sums.free)
    use = sums.n_kept >= 6
    Eu = np.asarray(edges)[use]
    N, Ta = sums.N[use], sums.T_a[use]
    R, p = Ta[:, :3, :3], Ta[:, :3, 3]
    ia = np.array([slot.get(int(a), F) for a in Eu[:, 0]])
    ib = np.array([slot.get(int(b), F) for b in Eu[:, 1]])
    G = []
    for c in (Eu[:, 0], Eu[:, 1]):
        Gc = np.zeros((len(Eu), 6, 6))
        Rt = np.transpose(R, (0, 2, 1))
        Gc[:, :3, :3] = Rt
        Gc[:, 3:, 3:] = Rt
        Gc[:, 3:, :3] = -Rt @ _skew(p - H0[c, :3, 3])
        G.append(Gc)
    rows, cols, vals = [], [], []
    r6, c6 = np.repeat(np.arange(6), 6), np.tile(np.arange(6), 6)
    for (i1, G1, s1) in ((ia, G[0], -1.0), (ib, G[1], 1.0)):
        for (i2, G2, s2) in ((ia, G[0], -1.0), (ib, G[1], 1.0)):
            ok = (i1 < F) & (i2 < F)
            B = s1 * s2 * np.transpose(G1, (0, 2, 1)) @ N @ G2
            rows.append((6 * i1[ok, None] + r6).ravel())
            cols.append((6 * i2[ok, None] + c6).ravel())
            vals.append(B[ok].reshape(-1, 36).ravel())
    if P_w is not None:
        for c, k in slot.items():
            rows.append(6 * k + np.arange(6))
            cols.append(6 * k + np.arange(6))
            vals.append(P_w[c])
    M = sparse.csc_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * F, 6 * F))
    lu = splu(M)
    from scipy.sparse.linalg import LinearOperator, eigsh
    lmax = eigsh(M, k=1, which="LA", return_eigenvectors=False)[0]
    inv = LinearOperator(M.shape, matvec=lu.solve, dtype=np.float64)
    lmin = 1.0 / eigsh(inv, k=1, which="LA", return_eigenvectors=False)[0]
    X = {}
    for c in set(sample) | {int(x) for a, b in Eu for x in (a, b) if a in slot and b in slot and
                            (a in sample or b in sample)}:
        rhs = np.zeros((6 * F, 6))
        rhs[6 * slot[c]:6 * slot[c] + 6] = np.eye(6)
        X[c] = lu.solve(rhs)

    def lever(c):
        Jm = np.eye(6)
        Jm[3:, :3] = -_skew(H[c][:3, 3] - H0[c][:3, 3])
        return Jm

    blk = lambda a, b: X[b][6 * slot[a]:6 * slot[a] + 6]  # (N'^-1)_ab, b sampled or a neighbour
    return slot, lever, blk, lmax / lmin


CAP = {"strip_1023": lambda: strip(1024, 20_000, 3_200), "strip_4095_priors": None,
       "block_32x32": lambda: _block(32), "block_64x64": lambda: _block(64)}


@pytest.mark.parametrize("problem", list(CAP))
def test_past_the_dense_cap_against_sparse_solves(eng, problem):
    """max_iterations=1: C_c / s0^2 of a seeded sample of 64 free clouds and the blocks of all their
    edges with two free ends against J' (N'^-1) J'^T from scipy's sparse LU of N'."""
    P = W = None
    if problem == "strip_4095_priors":
        scans, truth, H0, edges = strip(4096, 2_000, 12_800)
        P = _noisy(truth, 41, 0.03, 0.05)
        W = np.tile([0.01 ** 2 / np.deg2rad(0.03) ** 2] * 3 + [0.01 ** 2 / 0.05 ** 2] * 3, (4096, 1))
        H0 = P.copy()
    else:
        scans, truth, H0, edges = CAP[problem]()
    edges = np.asarray(edges)
    H, out = _joint(eng, 1, scans, edges, (0,), H0, P, W, max_iterations=1)
    cov, ecov, s0 = _sel(eng, len(scans), len(edges))
    sums = _oracle_sums(eng, scans, edges, H0)
    status = np.array([o.status for o in out])
    assert np.all(sums.n_kept[status != 0] < 6)
    rng = np.random.default_rng(7)
    sample = sorted(rng.choice(np.array(sums.free), 64, replace=False).tolist())
    slot, lever, blk, kappa = _sparse_reference(sums, edges, H0, H, sample, W)
    ku = kappa * np.finfo(np.float64).eps / 2
    sig_tol, corr_tol = max(10 * ku, 1e-12), max(100 * ku, 1e-12)
    d_sig = d_corr = 0.0
    for c in sample:
        ref = lever(c) @ blk(c, c) @ lever(c).T
        d_sig = max(d_sig, np.abs(_sig(cov[c] / s0 ** 2) / _sig(ref) - 1).max())
        d_corr = max(d_corr, np.abs(_corr(cov[c]) - _corr(ref)).max())
    # every edge of a sampled cloud with two free ends: its cross block through C_e
    n_edges_checked = 0
    for e, (a, b) in enumerate(edges):
        if a not in slot or b not in slot or not (a in sample or b in sample) or sums.n_kept[e] < 6:
            continue
        n_edges_checked += 1
        Ha = H[a]
        Ga, Gb = np.zeros((6, 6)), np.zeros((6, 6))
        Ga[:3, :3] = Ga[3:, 3:] = Gb[:3, :3] = Gb[3:, 3:] = Ha[:3, :3].T
        Ga[3:, :3] = -Ha[:3, :3].T @ _skew(H[b][:3, 3] - Ha[:3, 3])
        Ca, Cb = lever(a) @ blk(a, a) @ lever(a).T, lever(b) @ blk(b, b) @ lever(b).T
        Cab = lever(a) @ blk(a, b) @ lever(b).T
        M = Ga @ Cab @ Gb.T
        ref = Gb @ Cb @ Gb.T + Ga @ Ca @ Ga.T - M - M.T
        d_sig = max(d_sig, np.abs(_sig(ecov[e] / s0 ** 2) / _sig(ref) - 1).max())
        d_corr = max(d_corr, np.abs(_corr(ecov[e]) - _corr(ref)).max())
    print(f"{problem}: F={len(sums.free)}, 64 clouds and {n_edges_checked} edges, kappa u {ku:.1e}, "
          f"sigma rel {d_sig:.2e}, correlation abs {d_corr:.2e}")
    assert d_sig < sig_tol and d_corr < corr_tol


# --------------------------------------------------------------------------- structure, call order
def test_structure(eng):
    scans, truth, H0, edges = ring()
    clouds = list(scans) + [scans[3]]  # cloud 8: no edge references it
    H0x = np.concatenate([H0, H0[3:4]])
    _joint(eng, 1, clouds, edges, (0, 4), H0x)
    cov, ecov, s0 = _sel(eng, 9, len(edges))
    assert np.array_equal(cov[0], np.zeros((6, 6))) and np.array_equal(cov[4], np.zeros((6, 6)))
    assert np.isnan(cov[8]).all() and np.isfinite(cov[:8]).all() and np.isfinite(ecov).all()
    assert np.array_equal(cov, np.swapaxes(cov, 1, 2), equal_nan=True)
    assert np.array_equal(ecov, np.swapaxes(ecov, 1, 2))


def test_georeferenced_ring_gives_the_same_covariances(eng):
    """test_gpu_joint_cov's UTM test under the sparse solve: the ring with its world translated by
    (4.5e5, 5.4e6, 300), one iteration from the true poses; the local covariances, moved by the
    origin-based update's drift d_c as there, equal the UTM ones to 1e-6."""
    utm = np.array([4.5e5, 5.4e6, 300.0])
    scans, truth, H0, edges = ring()
    scans_u, truth_u, H0_u, _ = ring(shift=utm)
    p = _params(eng, max_iterations=1)
    fixed = np.zeros(len(scans), dtype=bool)
    fixed[0] = True
    eng.set_option("sign_mode", 1)
    eng.set_option("joint_solver", 1)
    try:
        H, _ = eng.register_joint(scans, edges, fixed, truth, 1000, 10, p, 1.0)
        cov, ecov, s0 = _sel(eng, len(scans), len(edges))
        H_u, _ = eng.register_joint(scans_u, edges, fixed, truth_u, 1000, 10, p, 1.0)
        cov_u, ecov_u, s0_u = _sel(eng, len(scans), len(edges))
    finally:
        eng.set_option("sign_mode", 0)
        eng.set_option("joint_solver", 0)
    drift = H_u[:, :3, 3] - utm - H[:, :3, 3]
    moved = np.array([_lever(d) @ C @ _lever(d).T for d, C in zip(drift, cov)])
    emoved = np.array([_lever(H[a][:3, :3].T @ drift[b]) @ C @ _lever(H[a][:3, :3].T @ drift[b]).T
                       for (a, b), C in zip(edges, ecov)])
    d_sig = max(np.abs(_sig(cov_u[1:]) / _sig(moved[1:]) - 1).max(), np.abs(_sig(ecov_u) / _sig(emoved) - 1).max())
    d_corr = max(np.abs(_corr(cov_u[1:]) - _corr(moved[1:])).max(), np.abs(_corr(ecov_u) - _corr(emoved)).max())
    print(f"georeferenced (sparse): drift {np.abs(drift).max():.1e} m, s0 rel {abs(s0_u / s0 - 1):.2e}, "
          f"sigma rel {d_sig:.2e}, correlation abs {d_corr:.2e}")
    assert abs(s0_u / s0 - 1) < 1e-6 and d_sig < 1e-6 and d_corr < 1e-6


def test_call_order_and_side_effects(eng):
    scans, truth, H0, edges = ring()
    p = _params(eng)
    n_c, n_e = len(scans), len(edges)
    X_fix, X_mov = _pair("bunny")
    eng.register_fused(X_fix, X_mov, 500, 10, 1.0, p)
    before = _one_pair_state(eng)
    H, out = _joint(eng, 1, scans, edges, (0,), H0)
    outs = eng.batch_outputs(out)
    a = _sel(eng, n_c, n_e)
    b = _sel(eng, n_c, n_e)
    assert _same_bits(a, b)
    for (x, r, lg, T), (x2, r2, lg2, T2) in zip(outs, eng.batch_outputs(out)):
        assert np.array_equal(x, x2) and np.array_equal(r, r2) and np.array_equal(T, T2)
        assert [bytes(g) for g in lg] == [bytes(g) for g in lg2]
    after = _one_pair_state(eng)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    # a following sparse call on this engine: the bits of a fresh engine
    H2, out2 = _joint(eng, 1, scans, edges, (0,), H0)
    c = _sel(eng, n_c, n_e)
    fresh = _capi.Engine(0)
    try:
        H3, out3 = _joint(fresh, 1, scans, edges, (0,), H0)
        f = fresh.joint_selected_covariances(n_c, n_e)
    finally:
        fresh.close()
    assert np.array_equal(H2, H3) and np.array_equal(H, H2) and _same_bits(c, f) and _same_bits(a, c)
    for nc, ne in ((n_c + 1, n_e), (n_c, n_e - 1)):
        with pytest.raises(SicpError) as ei:
            _sel(eng, nc, ne)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG
    # a later non-joint batched call
    eng.register_pairs(scans[:2], [(0, 1)], 1000, 10, p, 1.0)
    with pytest.raises(SicpError) as ei:
        _sel(eng, n_c, n_e)
    assert ei.value.code == _capi.SICP_ERR_STATE
    # a failed (singular) sparse call
    rng = np.random.default_rng(3)
    Pp = np.column_stack([rng.uniform(0, 10, (5000, 2)), np.zeros(5000)])
    Q = np.column_stack([rng.uniform(0, 10, (5000, 2)), np.zeros(5000)])
    _joint(eng, 1, scans, edges, (0,), H0)
    with pytest.raises(SicpError):
        _joint(eng, 1, [Pp, Q], [(0, 1)], (0,), None)
    with pytest.raises(SicpError) as ei:
        _sel(eng, 2, 1)
    assert ei.value.code == _capi.SICP_ERR_STATE


def test_simpleicp_joint_selected_on_a_strip_held_by_priors():
    scans, truth, H0, edges = strip(256, 20_000, 800)
    P = _noisy(truth, 51, 0.03, 0.05)
    W = np.tile([0.01 ** 2 / np.deg2rad(0.03) ** 2] * 3 + [0.01 ** 2 / 0.05 ** 2] * 3, (256, 1))
    kw = dict(fixed=(), H0=P, prior_poses=P, prior_weights=W, max_overlap_distance=1.0, max_iterations=10)
    s = sb.simpleicp_joint(scans, edges, solver="sparse", covariances="selected", **kw)
    d = sb.simpleicp_joint(scans, edges, solver="dense", covariances="selected", **kw)
    dt = sb.simpleicp_joint(scans, edges, solver="dense", covariances=True, **kw)
    assert _same_bits((d.cov, d.edge_cov, d.s0), (dt.cov, dt.edge_cov, dt.s0))
    assert np.isfinite(s.s0) and (np.einsum("cii->ci", s.cov) > 0).all()
    assert np.abs(_sig(s.cov) / _sig(d.cov) - 1).max() < 1e-6
    assert abs(s.s0 / d.s0 - 1) < 1e-9
