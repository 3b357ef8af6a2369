"""sicp_get_joint_covariances / simpleicp_joint(covariances=True) on the GPU: lock-step with the
NumPy statement of the rule (joint_cov_rule.py, which repeats the final iteration of the joint
restatement oracle/joint_oracle.py) on the ring and on strips of 127 and 255 free clouds, the
structure of the result (fixed, unused and shared clouds, duplicated edges, an edge without
overlap), georeferenced coordinates, the call order and the end-to-end call.

Tolerances against the oracle.  The lock-step tests of the registration prove that the device's
poses agree with the oracle's to 1e-9 (max |H| entry); in lock-step both sides take the same steps
from the same kept rows and float32 normals, so their residuals, and with them s0, differ by the
rounding of two float64 evaluations (s0 is asserted to 1e-12, and matches to ~1e-15).  N is summed
in a different order and parameterisation (the device centres about c_w, the oracle uses the world
origin), so its entries differ by a relative O(u), u = 1.1e-16, beyond what the pose difference
brings.  A relative change e of N changes N^-1 by up to kappa(N) e relative, and a 1e-9 pose
difference cannot reach e ~ 1e-9 without moving s0 far more than it does: e is rounding.  So
every sigma (square root of a variance) must agree to kappa u / 2, and a correlation rho =
C_ij / (s_i s_j), |rho| <= 1, to about 2 kappa u absolute.  Tolerances: SIG = 10 kappa u and
CORR = 100 kappa u with kappa the condition number of the rule's N (1e-12 at least).  On the ring
kappa ~ 1.5e6; a strip of 127 or 255 clouds chained along 250 to 510 m is far worse conditioned."""
import numpy as np
import pytest

import simpleicp_b200 as sb
from oracle import joint_oracle as J
from simpleicp_b200 import _capi
from simpleicp_b200._capi import SicpError

import joint_cov_rule as JC
from test_gpu_joint import _lockstep, _params, _pair, strip
from test_joint_host import ring

pytestmark = pytest.mark.gpu

S0_TOL = 1e-12  # s0 against the oracle and against the batch outputs' residuals


@pytest.fixture(scope="module")
def eng():
    e = _capi.Engine(0)
    yield e
    e.close()


def _sig(C):
    return np.sqrt(np.einsum("...ii->...i", C))


def _corr(C):
    s = _sig(C)
    return C / (s[..., :, None] * s[..., None, :])


def _s0_of_outputs(eng, out, F):
    ss, m = 0.0, 0
    for o, b in zip(out, eng.batch_outputs(out)):
        if b is not None:
            ss += float(b[1] @ b[1])
            m += b[1].size
    return np.sqrt(ss / (m - 6 * F))


def _compare(eng, out, ref, free, cov, ecov, s0):
    """ref: the rule's FinalIteration of the oracle run in lock-step with the device call `out`."""
    F = len(free)
    assert abs(s0 - _s0_of_outputs(eng, out, F)) <= S0_TOL * s0
    assert abs(s0 - ref.s0) <= S0_TOL * ref.s0, (s0, ref.s0)
    ku = np.linalg.cond(ref.N) * np.finfo(np.float64).eps / 2
    sig_tol, corr_tol = max(10 * ku, 1e-12), max(100 * ku, 1e-12)
    d_sig = max(np.abs(_sig(cov[free]) / _sig(ref.cov[free]) - 1).max(),
                np.abs(_sig(ecov) / _sig(ref.edge_cov) - 1).max())
    d_corr = max(np.abs(_corr(cov[free]) - _corr(ref.cov[free])).max(),
                 np.abs(_corr(ecov) - _corr(ref.edge_cov)).max())
    print(f"joint covariances F={F}: s0 {s0:.6e} rel {abs(s0 / ref.s0 - 1):.2e}, kappa u {ku:.1e}, "
          f"sigma rel {d_sig:.2e}, correlation abs {d_corr:.2e}")
    assert d_sig < sig_tol and d_corr < corr_tol, (d_sig, sig_tol, d_corr, corr_tol)


@pytest.mark.parametrize("problem", ["ring", "strip127", "strip255"])
def test_lockstep_with_the_oracle(eng, problem):
    if problem == "ring":
        scans, truth, H0, edges = ring()
        its = 30
    elif problem == "strip127":
        scans, truth, H0, edges = strip(128, 50_000, 400)
        its = 20
    else:  # the largest system: 255 free clouds, 1530 unknowns
        scans, truth, H0, edges = strip(256, 20_000, 800)
        its = 4
    H, out, logs, run = _lockstep(eng, scans, H0, edges, (0,), max_iterations=its)
    assert np.abs(H - run.H).max() < 1e-9
    ref = JC.final_iteration(scans, edges, run, H0=H0, max_overlap_distance=1.0)
    assert np.abs(ref.H - run.H).max() < 1e-12
    cov, ecov, s0 = eng.joint_covariances(len(scans), len(edges))
    free = np.arange(1, len(scans))
    _compare(eng, out, ref, free, cov, ecov, s0)
    assert np.array_equal(cov[0], np.zeros((6, 6)))


def test_structure(eng):
    """Fixed clouds 0 and 4, an unused cloud 6 (None), cloud 2 on both sides, edge (0, 1) twice and
    edge (0, 4) between two fixed clouds."""
    scans, truth, H0, edges = ring()
    p = _params(eng)
    clouds = list(scans[:6]) + [None]
    H0s = np.concatenate([H0[:6], np.eye(4)[None] * 2.0])
    E = np.array([(0, 1), (0, 1), (1, 2), (2, 3), (3, 4), (4, 5), (1, 3), (0, 4)])
    fixed = np.zeros(7, dtype=bool)
    fixed[[0, 4]] = True
    H, out = eng.register_joint(clouds, E, fixed, H0s, 1000, 10, p, 1.0)
    assert all(o.status == 0 for o in out)
    cov, ecov, s0 = eng.joint_covariances(7, len(E))
    assert np.array_equal(cov[0], np.zeros((6, 6))) and np.array_equal(cov[4], np.zeros((6, 6)))
    assert np.isnan(cov[6]).all()
    assert np.array_equal(ecov[7], np.zeros((6, 6)))  # (0, 4): both fixed
    assert np.array_equal(ecov[0], ecov[1])            # the duplicate
    Gb = np.zeros((6, 6))
    Gb[:3, :3] = Gb[3:, 3:] = H[0][:3, :3].T
    assert np.abs(ecov[0] - Gb @ cov[1] @ Gb.T).max() <= 1e-12 * np.abs(ecov[0]).max()
    for c in (1, 2, 3, 5):
        assert np.array_equal(cov[c], cov[c].T) and np.linalg.eigvalsh(cov[c]).min() > 0
    # against the oracle with the device's normals
    from test_gpu_joint import _device_normals
    nrm_ref = J.simpleicp_joint(clouds, E, fixed=(0, 4), H0=H0s, max_iterations=0, max_overlap_distance=1.0)
    nrm = {e: _device_normals(eng, clouds[a], nrm_ref.idx_fix[e]) for e, (a, _) in enumerate(E)}
    run = J.simpleicp_joint(clouds, E, fixed=(0, 4), H0=H0s, max_iterations=30, max_overlap_distance=1.0,
                            normals=nrm)
    ref = JC.final_iteration(clouds, E, run, fixed=(0, 4), H0=H0s, max_overlap_distance=1.0)
    assert np.abs(ref.H - run.H).max() < 1e-12
    H2, out2 = eng.register_joint(clouds, E, fixed, H0s, 1000, 10, p, 1.0)
    cov2, ecov2, s02 = eng.joint_covariances(7, len(E))
    assert np.array_equal(cov, cov2, equal_nan=True) and np.array_equal(ecov, ecov2) and s0 == s02
    free = np.array([1, 2, 3, 5])
    ecov_free = np.delete(ecov, 7, axis=0)
    ref.edge_cov = np.delete(ref.edge_cov, 7, axis=0)
    _compare(eng, out2, ref, free, cov, ecov_free, s0)


def test_an_edge_without_overlap_gets_a_covariance_from_the_poses(eng):
    """The configuration of test_gpu_joint's failures: edge (0, 3) has no overlap and takes no part;
    its covariance is G_b C_3 G_b^T (cloud 0 is fixed) at the returned poses."""
    scans, truth, H0, edges = ring()
    p = _params(eng)
    W7 = scans[7] @ truth[7][:3, :3].T + truth[7][:3, 3]
    tail = np.ascontiguousarray(scans[7][W7[:, 0] >= 28.0])
    c4 = [scans[0], scans[2], scans[4], tail]
    H04 = np.stack([H0[0], H0[2], H0[4], H0[7]])
    H, out = eng.register_joint(c4, [(0, 1), (1, 2), (2, 3), (0, 3)], np.array([True, False, False, False]), H04,
                                1000, 10, p, 1.0)
    assert out[3].status == _capi.SICP_ERR_NO_OVERLAP
    cov, ecov, s0 = eng.joint_covariances(4, 4)
    Gb = np.zeros((6, 6))
    Gb[:3, :3] = Gb[3:, 3:] = H[0][:3, :3].T
    assert np.isfinite(ecov[3]).all()
    assert np.abs(ecov[3] - Gb @ cov[3] @ Gb.T).max() <= 1e-12 * np.abs(ecov[3]).max()
    assert abs(s0 - _s0_of_outputs(eng, out, 3)) <= 1e-12 * s0


def _lever(d):
    M = np.eye(6)
    M[3:, :3] = -J.skew(d)
    return M


def test_georeferenced_ring_gives_the_same_covariances(eng):
    """The ring with its world translated by (4.5e5, 5.4e6, 300): the same scans in their own
    frames, the poses moved; one iteration from the true poses.  N is centred about c_w and every
    lever arm is a difference of positions, so the device arithmetic depends on the translation only
    through rounding.  One effect is not rounding: the origin-based update moves the returned UTM
    origins by about |alpha|^2 D (DESIGN.md §6.9) against the local ones, d_c = o_c^utm - utm - o_c.
    Moving the point whose displacement u_c describes by d_c maps u_c by J(d_c) = [[I, 0],
    [-[d_c]x, I]], and u_e by J(R_a^T d_b) (cloud b's origin in frame a), so the local covariances,
    mapped so, must equal the UTM ones.  Tolerance: the shifted generator's scans differ by up to
    3e-9 m (the ulp of 5.4e6 m) against residuals of ~7e-3 m, at most 4e-7 relative per residual
    and incoherent over the rows; every sigma and s0 to 1e-6 relative, correlations to 1e-6."""
    utm = np.array([4.5e5, 5.4e6, 300.0])
    scans, truth, H0, edges = ring()
    scans_u, truth_u, H0_u, _ = ring(shift=utm)
    p = _params(eng, max_iterations=1)
    fixed = np.zeros(len(scans), dtype=bool)
    fixed[0] = True
    eng.set_option("sign_mode", 1)
    try:
        H, _ = eng.register_joint(scans, edges, fixed, truth, 1000, 10, p, 1.0)
        cov, ecov, s0 = eng.joint_covariances(len(scans), len(edges))
        H_u, _ = eng.register_joint(scans_u, edges, fixed, truth_u, 1000, 10, p, 1.0)
        cov_u, ecov_u, s0_u = eng.joint_covariances(len(scans), len(edges))
    finally:
        eng.set_option("sign_mode", 0)
    drift = H_u[:, :3, 3] - utm - H[:, :3, 3]
    moved = np.array([_lever(d) @ C @ _lever(d).T for d, C in zip(drift, cov)])
    emoved = np.array([_lever(H[a][:3, :3].T @ drift[b]) @ C @ _lever(H[a][:3, :3].T @ drift[b]).T
                       for (a, b), C in zip(edges, ecov)])
    d_sig = max(np.abs(_sig(cov_u[1:]) / _sig(moved[1:]) - 1).max(), np.abs(_sig(ecov_u) / _sig(emoved) - 1).max())
    d_corr = max(np.abs(_corr(cov_u[1:]) - _corr(moved[1:])).max(), np.abs(_corr(ecov_u) - _corr(emoved)).max())
    print(f"georeferenced: drift {np.abs(drift).max():.1e} m, s0 rel {abs(s0_u / s0 - 1):.2e}, "
          f"sigma rel {d_sig:.2e}, correlation abs {d_corr:.2e}")
    assert abs(s0_u / s0 - 1) < 1e-6 and d_sig < 1e-6 and d_corr < 1e-6


def _one_pair_state(eng):
    import ctypes as C
    res = np.empty(4096)
    n = C.c_int64(0)
    eng._check(eng._lib.sicp_get_residuals(eng._h, res.ctypes.data, res.size, C.byref(n)))
    return eng.get_transform(), res[:n.value].copy()


def test_call_order(eng):
    scans, truth, H0, edges = ring()
    p = _params(eng)
    fixed = np.zeros(len(scans), dtype=bool)
    fixed[0] = True
    n_c, n_e = len(scans), len(edges)

    def state_error(code=_capi.SICP_ERR_STATE, nc=n_c, ne=n_e):
        with pytest.raises(SicpError) as ei:
            eng.joint_covariances(nc, ne)
        assert ei.value.code == code

    def joint():
        return eng.register_joint(scans, edges, fixed, H0, 1000, 10, p, 1.0)

    fresh = _capi.Engine(0)  # nothing yet
    try:
        with pytest.raises(SicpError) as ei:
            fresh.joint_covariances(n_c, n_e)
        assert ei.value.code == _capi.SICP_ERR_STATE
    finally:
        fresh.close()
    X_fix, X_mov = _pair("bunny")
    eng.register_fused(X_fix, X_mov, 500, 10, 1.0, p)
    before = _one_pair_state(eng)
    eng.set_map(scans[0])
    H, out = joint()
    outs = eng.batch_outputs(out)
    a = eng.joint_covariances(n_c, n_e)
    b = eng.joint_covariances(n_c, n_e)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a[:2], b[:2])) and a[2] == b[2]
    # the get changes neither the batch outputs, nor the map, nor the one-pair state
    for (x, r, lg, T), (x2, r2, lg2, T2) in zip(outs, eng.batch_outputs(out)):
        assert np.array_equal(x, x2) and np.array_equal(r, r2) and np.array_equal(T, T2)
        assert [bytes(g) for g in lg] == [bytes(g) for g in lg2]
    assert np.array_equal(eng.get_map(), scans[0])
    after = _one_pair_state(eng)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    # a second identical call: the same bits
    joint()
    c = eng.joint_covariances(n_c, n_e)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a[:2], c[:2])) and a[2] == c[2]
    state_error(_capi.SICP_ERR_BAD_ARG, nc=n_c + 1)
    state_error(_capi.SICP_ERR_BAD_ARG, ne=n_e - 1)
    # every call that replaces or clears the batch outputs
    for other in (lambda: eng.register_pairs(scans[:2], [(0, 1)], 1000, 10, p, 1.0),
                  lambda: eng.register_batch([(scans[0], scans[1])], 1000, 10, p, 1.0),
                  lambda: eng.register_to_map([scans[1]], 1000, 10, p, 1.0),
                  lambda: eng.map_insert([scans[1]], voxel_size=0.5),
                  lambda: eng.set_map(scans[0])):
        joint()
        eng.joint_covariances(n_c, n_e)
        other()
        state_error()
    # a failed joint call: two clouds sampled from one plane, a singular joint matrix
    joint()
    rng = np.random.default_rng(3)
    P = np.column_stack([rng.uniform(0, 10, (5000, 2)), np.zeros(5000)])
    Q = np.column_stack([rng.uniform(0, 10, (5000, 2)), np.zeros(5000)])
    with pytest.raises(SicpError):
        eng.register_joint([P, Q], [(0, 1)], np.array([True, False]), None, 1000, 10, p, 1.0)
    state_error(nc=2, ne=1)
    eng.set_map(None)


def test_simpleicp_joint_end_to_end():
    scans, truth, H0, edges = ring()
    res = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0, covariances=True)
    assert res.cov.shape == (8, 6, 6) and res.edge_cov.shape == (len(edges), 6, 6) and res.s0 > 0
    for c in range(1, 8):
        assert np.array_equal(res.cov[c], res.cov[c].T) and np.linalg.eigvalsh(res.cov[c]).min() > 0
    for e in range(len(edges)):
        assert np.linalg.eigvalsh(res.edge_cov[e]).min() > 0
    # cloud 0 is fixed; 1, 2 and 7 share an edge with it, 3 .. 6 are two edges away
    pos = np.sqrt(np.trace(res.cov[:, 3:, 3:], axis1=1, axis2=2))
    assert pos[3:7].max() > pos[[1, 2, 7]].max()
    default = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0)
    assert default.cov is None and default.edge_cov is None and default.s0 is None
    assert np.array_equal(default.H, res.H)
