"""Host-side tests of the a-posteriori covariances of the joint registration (DESIGN.md §6.9): the
NumPy statement of the rule (joint_cov_rule.py, over the joint restatement oracle/joint_oracle.py)
repeating the oracle's final iteration faithfully, against a direct statement on one edge, the
edge covariance under swapped roles, s0 against the noise of the scans, and the argument check of
simpleicp_joint(covariances=)."""
import numpy as np
import pytest

import simpleicp_b200 as sb
from oracle import joint_oracle as J

import joint_cov_rule as JC
from test_gpu_joint import strip
from test_joint_host import _clouds, _pair, ring


def _rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def test_one_edge_equals_s0_squared_j_inverse_normal_matrix_j():
    """Two clouds, one edge, cloud 0 fixed at I: frame a is the world and the joint matrix is A^T A
    of the final kept rows, so C_1 = s0^2 J (A^T A)^-1 J^T with s0^2 = |A xi - l|^2 / (n - 6) and
    J = [[I, 0], [-[o_1]x, I]] at the returned origin o_1."""
    X_fix, X_mov = _pair("dragon")
    res = J.simpleicp_joint([X_fix, X_mov], [(0, 1)], fixed=(0,), max_iterations=30)
    fi = JC.final_iteration([X_fix, X_mov], [(0, 1)], res, max_iterations=30)
    # the repeated final iteration is the oracle's
    assert np.abs(fi.H - res.H).max() < 1e-12
    assert np.abs(fi.xi[0] - res.log[-1][0].xi).max() <= 1e-12 * np.abs(res.log[-1][0].xi).max()
    assert fi.A[0].shape[0] == res.log[-1][0].n_kept
    res = fi
    A, l, xi = fi.A[0], fi.l[0], fi.xi[0]
    r = A @ xi - l
    s0sq = float(r @ r) / (A.shape[0] - 6)
    Jm = np.eye(6)
    Jm[3:, :3] = -J.skew(res.H[1][:3, 3])
    C = s0sq * Jm @ np.linalg.inv(A.T @ A) @ Jm.T
    assert _rel(res.cov[1], C) < 1e-12
    assert abs(res.s0 - np.sqrt(s0sq)) <= 1e-12 * np.sqrt(s0sq)
    assert np.array_equal(res.cov[0], np.zeros((6, 6)))
    # edge (0, 1) with a fixed at I: G_b = I
    assert _rel(res.edge_cov[0], C) < 1e-12


def test_swapped_roles_map_through_the_inverse_relative_pose():
    """Edges (2, 3) and (3, 2) of one adjustment: u_(3,2) = K u_(2,3) with R = R_23, q = q_23 and
    K = [[-R^T, 0], [-R^T [q]x, -R^T]] (the first-order change of the inverse relative pose), an
    identity of the linear propagation, so C_(3,2) = K C_(2,3) K^T to rounding."""
    scans, truth, H0, edges = ring()
    E = np.concatenate([edges, [(3, 2)]])
    ref = J.simpleicp_joint(scans, E, fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0)
    res = JC.final_iteration(scans, E, ref, H0=H0, max_overlap_distance=1.0)
    assert np.abs(res.H - ref.H).max() < 1e-12
    e23 = [k for k, (a, b) in enumerate(E) if (a, b) == (2, 3)][0]
    R23 = np.linalg.inv(res.H[2]) @ res.H[3]
    R, q = R23[:3, :3], R23[:3, 3]
    K = np.zeros((6, 6))
    K[:3, :3] = -R.T
    K[3:, 3:] = -R.T
    K[3:, :3] = -R.T @ J.skew(q)
    assert _rel(res.edge_cov[-1], K @ res.edge_cov[e23] @ K.T) < 1e-9
    # every free cloud: symmetric positive definite
    for c in range(1, len(scans)):
        assert np.allclose(res.cov[c], res.cov[c].T, rtol=0, atol=1e-12 * np.abs(res.cov[c]).max())
        assert np.linalg.eigvalsh(res.cov[c]).min() > 0


@pytest.mark.parametrize("problem", ["ring", "strip"])
def test_s0_matches_the_point_to_plane_noise(problem):
    """Every point carries Gaussian noise of sigma per coordinate (ring: isotropic, 5 mm) or along
    world z (strip: 1 cm, on a surface whose normals lie within about 20 degrees of z).  A
    point-to-plane residual n . (p_b - p_a) takes the noise of both points, so its standard
    deviation is about sqrt(2) sigma (times |n_z| ~ 0.95 for the strip).  s0 lands within a factor
    1.2 of that (measured: 1.01 on both): the 3-sigma rejection trims the tails, the
    nearest-neighbour match prefers points whose noise brings them closer, the float normals of
    noisy neighbourhoods tilt a little and the surface curves within a neighbourhood -- shifts of a
    few per cent each, none near 20 %."""
    if problem == "ring":
        scans, truth, H0, edges = ring()
        expect = np.sqrt(2.0) * 0.005
    else:
        scans, truth, H0, edges = strip(8, 20_000, 16)
        expect = np.sqrt(2.0) * 0.01 * 0.95
    ref = J.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0)
    res = JC.final_iteration(scans, edges, ref, H0=H0, max_overlap_distance=1.0)
    assert expect / 1.2 < res.s0 < expect * 1.2, (res.s0, expect)


@pytest.mark.parametrize("value", [1, 0, "yes", None, 1.0, np.array([True])])
def test_covariances_must_be_a_bool(value):
    with pytest.raises(TypeError, match="covariances"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], covariances=value)
