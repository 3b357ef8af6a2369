"""Host-side tests of the joint registration with pose priors (DESIGN.md §6.12): simpleicp_joint's
argument checks, the C ABI declaration of sicp_register_joint_priors, and the NumPy restatement
with priors (joint_prior_oracle.py, on top of oracle/joint_oracle.py): zero weights, the first step
against a direct solve, a huge weight against a fixed cloud, a ring anchored by a prior alone, and
the s0 rule with priors."""
import re
from pathlib import Path

import numpy as np
import pytest

import simpleicp_b200 as sb
from oracle import joint_oracle as J
from simpleicp_b200 import _capi
from simpleicp_b200.batch import _joint_priors

import joint_cov_rule
import joint_prior_cov_rule
import joint_prior_oracle as JPO
from test_joint_host import ring

REPO = Path(__file__).resolve().parents[1]


def _clouds(n=3, m=200):
    rng = np.random.default_rng(1)
    return [rng.normal(size=(m, 3)) for _ in range(n)]


def _eye(n=3):
    return np.tile(np.eye(4), (n, 1, 1))


def _w(n=3, v=1.0):
    return np.full((n, 6), v)


def _set(a, idx, v):
    a = a.copy()
    a[idx] = v
    return a


@pytest.mark.parametrize("kw,msg", [
    ({"prior_poses": _eye()}, "given together"),
    ({"prior_weights": _w()}, "given together"),
    ({"prior_poses": _eye(2), "prior_weights": _w()}, r"prior_poses must have shape \(3, 4, 4\)"),
    ({"prior_poses": _eye(), "prior_weights": _w(3)[:, :5]}, r"prior_weights must have shape \(3, 6\)"),
    ({"prior_poses": _eye(), "prior_weights": _set(_w(), (1, 2), -1.0)}, "finite and >= 0"),
    ({"prior_poses": _eye(), "prior_weights": _set(_w(), (1, 4), np.nan)}, "finite and >= 0"),
    ({"prior_poses": _eye(), "prior_weights": _set(_w(), (1, 0), np.inf)}, "finite and >= 0"),
    # a weight of a cloud whose prior is not read is checked all the same
    ({"prior_poses": _eye(), "prior_weights": _set(_w(), (0, 0), -1.0)}, "finite and >= 0"),
    ({"prior_poses": _set(_eye(), (1, 0, 3), np.nan), "prior_weights": _w()}, r"prior_poses\[1\] has non-finite"),
    ({"prior_poses": _set(_eye(), (1, 0, 0), 1.0 + 1e-5), "prior_weights": _w()}, "orthonormal"),
    ({"prior_poses": _set(_eye(), (1, 3, 0), 1e-3), "prior_weights": _w()}, "bottom row"),
    # fixed=() is legal with priors, but a position-only prior does not anchor
    ({"fixed": (), "prior_poses": _eye(), "prior_weights": _set(_w(), (slice(None), slice(0, 3)), 0.0)},
     "no path to a fixed cloud over the edges and no pose prior with six non-zero weights"),
    ({"fixed": (), "prior_poses": _eye(), "prior_weights": _w(v=0.0)}, "no path to a fixed cloud"),
])
def test_prior_argument_checks(kw, msg):
    with pytest.raises(ValueError, match=msg):
        sb.simpleicp_joint(_clouds(), [(0, 1), (1, 2)], **kw)


def test_without_priors_the_messages_are_unchanged():
    with pytest.raises(ValueError, match=r"^fixed must be a sequence of at least one integer cloud index$"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], fixed=())
    with pytest.raises(ValueError, match=r"^free cloud 1 has no path to a fixed cloud over the edges$"):
        sb.simpleicp_joint(_clouds(), [(1, 2)])


def test_priors_that_are_not_read_may_hold_nan():
    """Cloud 0 is fixed, cloud 2 has zero weights and cloud 3 no edge: their poses are not read.
    Cloud 1's full prior anchors; a rotation inside 1e-6 of orthonormal passes."""
    free = np.array([False, True, True, False])
    P = _eye(4)
    P[[0, 2, 3]] = np.nan
    P[1, :3, :3] *= 1.0 + 4e-7
    W = np.ones((4, 6))
    W[2] = 0.0
    Pc, Wc, full = _joint_priors(P, W, free)
    assert list(full) == [False, True, False, False]
    assert Pc.dtype == Wc.dtype == np.float64
    W[1, 3:] = 0.0
    assert list(_joint_priors(P, W, free)[2]) == [False] * 4  # rotation only: read, not an anchor


def test_abi_declares_the_prior_entry_point():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    decl = re.search(r"int32_t sicp_register_joint_priors\(([^;]*)\);", header)
    assert decl and "sicp_register_joint_priors" in _capi.SYMBOLS
    params = re.sub(r"/\*.*?\*/", "", decl.group(1)).split(",")
    assert len(params) == 15
    assert [p.split()[-1] for p in params[9:11]] == ["prior_H", "prior_w"]


def _noisy_priors(truth, seed, rot_deg=0.02, pos_m=0.03):
    rng = np.random.default_rng(seed)
    P = []
    for T in truth:
        dx = np.concatenate((np.deg2rad(rng.normal(0, rot_deg, 3)), rng.normal(0, pos_m, 3)))
        R = J.rigid_from_x(dx)
        U, _, Vt = np.linalg.svd(R[:3, :3])  # rigid_from_x is rigid; the SVD only states it
        R[:3, :3] = U @ Vt
        P.append(R @ T)
    return np.array(P)


def test_oracle_zero_weights_give_the_result_without_priors_bit_for_bit():
    scans, truth, H0, edges = ring()
    kw = dict(fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0)
    ref = J.simpleicp_joint(scans, edges, **kw)
    P = np.full((8, 4, 4), np.nan)
    for solver in ("dense", "sparse"):
        a = J.simpleicp_joint(scans, edges, solver=solver, **kw)
        for b in (JPO.simpleicp_joint(scans, edges, solver=solver, **kw),
                  JPO.simpleicp_joint(scans, edges, solver=solver, prior_poses=P, prior_weights=np.zeros((8, 6)), **kw)):
            assert np.array_equal(a.H, b.H) and len(a.log) == len(b.log) and a.converged == b.converged
            for ra, rb in zip(a.log, b.log):
                assert [e.n_kept for e in ra] == [e.n_kept for e in rb]
                assert [(e.mean, e.std) for e in ra] == [(e.mean, e.std) for e in rb]
                assert all(np.array_equal(ea.xi, eb.xi) for ea, eb in zip(ra, rb) if ea.xi is not None)
    assert np.array_equal(ref.H, J.simpleicp_joint(scans, edges, solver="dense", **kw).H)


def _rotvec(R):
    """The rotation vector of a rotation by less than pi, from the trace and the skew part."""
    th = np.arccos(np.clip((np.trace(R) - 1.0) / 2.0, -1.0, 1.0))
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return v * (0.5 if th == 0.0 else th / (2.0 * np.sin(th)))


def test_oracle_first_step_is_the_direct_solve_with_the_prior_blocks():
    """The first step with priors (full on clouds 2 and 5, position only on 3 and 6) equals a solve
    of first_iteration_sums' system plus the stated blocks J^T W J and right-hand sides J^T W l,
    with J = [[I, 0], [-[o_c]x, I]] and l = (rotvec(R_P R_c^T), o_P - o_c) at H0."""
    scans, truth, H0, edges = ring()
    P = _noisy_priors(truth, 5)
    W = np.zeros((8, 6))
    W[[2, 5]] = [400.0, 400.0, 400.0, 25.0, 25.0, 25.0]
    W[[3, 6], 3:] = [9.0, 16.0, 4.0]
    ref = JPO.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_iterations=1, max_overlap_distance=1.0,
                              prior_poses=P, prior_weights=W)
    s = J.first_iteration_sums(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0)
    M, g = np.zeros((42, 42)), np.zeros(42)
    for (a, b), N, h, Ta in zip(edges, s.N, s.g, s.T_a):
        Ad = J.ad_world_to_frame(Ta)
        for c, sgn in ((a, -1.0), (b, 1.0)):
            if c > 0:
                i = 6 * (c - 1)
                g[i:i + 6] += sgn * Ad.T @ h
                for d, sgn2 in ((a, -1.0), (b, 1.0)):
                    if d > 0:
                        j = 6 * (d - 1)
                        M[i:i + 6, j:j + 6] += sgn * sgn2 * Ad.T @ N @ Ad
    for c in (2, 3, 5, 6):
        Jc = np.eye(6)
        Jc[3:, :3] = -J.skew(H0[c][:3, 3])
        l = np.concatenate((_rotvec(P[c][:3, :3] @ H0[c][:3, :3].T), P[c][:3, 3] - H0[c][:3, 3]))
        i = 6 * (c - 1)
        M[i:i + 6, i:i + 6] += Jc.T @ np.diag(W[c]) @ Jc
        g[i:i + 6] += Jc.T @ (W[c] * l)
    x = np.linalg.solve(M, g)
    for c in range(1, 8):
        H = J.rigid_from_x(x[6 * (c - 1):6 * c]) @ H0[c]
        assert np.abs(H - ref.H[c]).max() <= 1e-12 * np.abs(H).max()


def test_oracle_huge_weight_equals_a_fixed_cloud():
    """Weights w = 1e12 on all six components of cloud 3 with P_3 = H0[3] against cloud 3 in fixed.
    The prior leaves cloud 3 an increment of about |N_33| |x| / w per iteration (N_33 its block of the
    joint matrix without the prior, |x| the increments of its neighbours), and the other clouds follow
    it by at most as much.  |N| over the first iteration is about 1e5 and |x| below 0.1, so the poses
    may differ by about 1e-8 per iteration; over 30 iterations the bound below, 1e3 |N| / w, keeps a
    margin of 30.  The kept counts are equal in every iteration."""
    scans, truth, H0, edges = ring()
    kw = dict(H0=H0, max_iterations=30, max_overlap_distance=1.0)
    fixed = J.simpleicp_joint(scans, edges, fixed=(0, 3), **kw)
    W = np.zeros((8, 6))
    W[3] = 1e12
    pri = JPO.simpleicp_joint(scans, edges, fixed=(0,), prior_poses=H0, prior_weights=W, **kw)
    s = J.first_iteration_sums(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0)
    Nnorm = max(np.linalg.norm(J.ad_world_to_frame(Ta).T @ N @ J.ad_world_to_frame(Ta), 2)
                for N, Ta in zip(s.N, s.T_a))
    assert 1e4 < Nnorm < 1e6
    tol = 1e3 * Nnorm / 1e12
    assert len(pri.log) == len(fixed.log)
    for ra, rb in zip(pri.log, fixed.log):
        assert [e.n_kept for e in ra] == [e.n_kept for e in rb]
    assert np.abs(pri.H - fixed.H).max() < tol


def test_oracle_ring_anchored_by_one_prior_alone_converges():
    """fixed=(): cloud 0's full prior at its true pose anchors the ring."""
    scans, truth, H0, edges = ring()
    W = np.zeros((8, 6))
    W[0] = 1e4
    for solver in ("dense", "sparse"):
        res = JPO.simpleicp_joint(scans, edges, fixed=(), H0=H0, max_iterations=30, max_overlap_distance=1.0,
                                prior_poses=truth, prior_weights=W, solver=solver)
        assert res.converged
        assert np.abs(res.H - truth).max() < 1e-2


def test_s0_rule_with_priors():
    """The restatement with priors: zero weights give joint_cov_rule's s0 and covariances; with
    priors s0 counts their residuals and weights, and removing their blocks from N grows no
    diagonal entry of N^-1."""
    scans, truth, H0, edges = ring()
    kw = dict(fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0)
    res = J.simpleicp_joint(scans, edges, **kw)
    base = joint_cov_rule.final_iteration(scans, edges, res, **kw)
    zero = joint_prior_cov_rule.final_iteration(scans, edges, res, prior_poses=np.full((8, 4, 4), np.nan),
                                                prior_weights=np.zeros((8, 6)), **kw)
    assert np.array_equal(zero.N, base.N) and zero.s0 == base.s0 and np.array_equal(zero.cov, base.cov)
    P = _noisy_priors(truth, 7)
    W = np.zeros((8, 6))
    W[[2, 5]] = 1e3
    W[[4, 7], 3:] = 1e3
    resp = JPO.simpleicp_joint(scans, edges, prior_poses=P, prior_weights=W, **kw)
    fi = joint_prior_cov_rule.final_iteration(scans, edges, resp, prior_poses=P, prior_weights=W, **kw)
    assert np.abs(fi.H - resp.H).max() < 1e-12
    m = sum(a.shape[0] for a in fi.A if a.shape[0] >= 6) + 2 * 6 + 2 * 3
    assert np.isfinite(fi.s0) and m > 42
    N0 = fi.N.copy()
    for p in fi.priors:
        N0[6 * p.slot:6 * p.slot + 6, 6 * p.slot:6 * p.slot + 6] -= p.N
    d_base = np.diagonal(np.linalg.inv(N0))
    d_pri = np.diagonal(np.linalg.inv(fi.N))
    assert (d_pri <= d_base * (1 + 1e-12)).all() and (d_pri < d_base * 0.999).any()
